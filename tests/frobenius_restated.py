"""Exact restatement of the Frobenius ground truth (frob_pass_kernel / frob_compact_kernel / reproject_lafs_kernel in
affnet_b200/csrc/verify.cu), operation by operation, in numpy (test infrastructure, not product).

float64 steps are numpy float64 operations in the kernel's order (verify.cu is built without fused multiply-adds); fp32 steps are
numpy float32 operations, each correctly rounded and never fused; the one fused multiply-add (the centre distance's dot, shared with
gt_kernel) is `scale_space_restated.fmaf32`.  So a kernel that differs from these functions in one bit is wrong.

Next to it, `d_bound` is the per-element bound within which the reference's fp32 distances (torch.inverse, bmm, an fp32 H^-1) and these
agree; DESIGN.md states its derivation."""
import numpy as np

from scale_space_restated import fmaf32

F = np.float32
U32 = 2.0 ** -24
K_STEPS = 64          # rounding steps charged to each entry of E = B A' - I and r = B t' + c on either side (DESIGN.md)


class Params:
    """ag_frobenius_params_t."""

    def __init__(self, dist_threshold=4.0, center_dist_th=None, scale_diff_coef=0.3, skip_center=False, do_up_is_up=False, inv_to_eye=True):
        self.th = F(dist_threshold)
        self.gate = center_dist_th is not None
        self.cth = F(center_dist_th if self.gate else 0.0)
        self.coef = F(scale_diff_coef)
        self.skip, self.up, self.inv = bool(skip_center), bool(do_up_is_up), bool(inv_to_eye)


def inverse_h(H):
    """inverse_h: adj(H) / det(H) of the fp32 H in float64 (adj3's order) -> [9]."""
    H = np.asarray(H, F).astype(np.float64).reshape(9)
    m = H
    A = np.array([m[4] * m[8] - m[5] * m[7], m[2] * m[7] - m[1] * m[8], m[1] * m[5] - m[2] * m[4],
                  m[5] * m[6] - m[3] * m[8], m[0] * m[8] - m[2] * m[6], m[2] * m[3] - m[0] * m[5],
                  m[3] * m[7] - m[4] * m[6], m[1] * m[6] - m[0] * m[7], m[0] * m[4] - m[1] * m[3]])
    with np.errstate(all="ignore"):
        det = H[0] * A[0] + H[1] * A[3] + H[2] * A[6]
        return A / det


def rectify32(a00, a01, a10, a11):
    """rectify_up_is_up (common.cuh) in fp32."""
    with np.errstate(all="ignore"):
        det = np.sqrt(np.abs((a00 * a11 - a10 * a01) + F(1e-10)))
        b2a2 = np.sqrt(a01 * a01 + a00 * a00)
        return b2a2 / det, F(0.0) * det, (a11 * a01 + a10 * a00) / (b2a2 * det), det / b2a2


def frame_2x2(a, up):
    """frame_2x2: s = sqrt|det A| (float64, rounded once) and, with up, A <- rectify(A / s) s in fp32.  a [n,4] fp32."""
    a = [np.asarray(a[:, k], F) for k in range(4)]
    d = [x.astype(np.float64) for x in a]
    with np.errstate(all="ignore"):
        s = np.sqrt(np.abs(d[0] * d[3] - d[1] * d[2])).astype(F)
        if up:
            r = rectify32(a[0] / s, a[1] / s, a[2] / s, a[3] / s)
            a = [x * s for x in r]
    return np.stack(a, 1).astype(F), s


def reproject(lafs, G):
    """reproject_laf through G (float64 [9]) of lafs [n,2,3] -> (A' [n,4] fp32 row-major, t' [n,2] fp32)."""
    l = np.asarray(lafs, F).reshape(-1, 6).astype(np.float64)
    x, y = l[:, 2], l[:, 5]
    with np.errstate(all="ignore"):
        w = G[6] * x + G[7] * y + G[8]
        n1 = G[0] * x + G[1] * y + G[2]
        n2 = G[3] * x + G[4] * y + G[5]
        q1, q2 = n1 / (w * w), n2 / (w * w)
        j00, j01 = G[0] / w - q1 * G[6], G[1] / w - q1 * G[7]
        j10, j11 = G[3] / w - q2 * G[6], G[4] / w - q2 * G[7]
        a00, a01, a10, a11 = l[:, 0], l[:, 1], l[:, 3], l[:, 4]
        A = np.stack([j00 * a00 + j01 * a10, j00 * a01 + j01 * a11, j10 * a00 + j11 * a10, j10 * a01 + j11 * a11], 1).astype(F)
        t = np.stack([n1 / w, n2 / w], 1).astype(F)
    return A, t


def reproject_lafs(lafs, H, invert, up):
    """ag_reproject_lafs of one set -> [n,2,3] fp32."""
    G = inverse_h(H) if invert else np.asarray(H, F).astype(np.float64).reshape(9)
    A, t = reproject(lafs, G)
    A, _ = frame_2x2(A, up)
    return np.stack([A[:, 0], A[:, 1], t[:, 0], A[:, 2], A[:, 3], t[:, 1]], 1).reshape(-1, 2, 3)


def _sq_norm64(A, t, skip):
    q = A[:, 0].astype(np.float64) ** 2
    for k in range(1, 4):
        q = q + A[:, k].astype(np.float64) * A[:, k].astype(np.float64)
    if not skip:
        q = q + t[:, 0].astype(np.float64) * t[:, 0].astype(np.float64) + t[:, 1].astype(np.float64) * t[:, 1].astype(np.float64) + 1.0
    return q.astype(F)


def rows(lafs1, prm):
    """frob_row of lafs1 [n,2,3] -> dict of fp32 arrays."""
    l = np.asarray(lafs1, F).reshape(-1, 6)
    a, s = frame_2x2(l[:, [0, 1, 3, 4]], prm.up)
    x, y = l[:, 2].copy(), l[:, 5].copy()
    r = dict(x=x, y=y, na=x * x + y * y, s1e=s + F(1e-12), s=s)
    if prm.inv:
        d = a.astype(np.float64)
        with np.errstate(all="ignore"):
            det = d[:, 0] * d[:, 3] - d[:, 1] * d[:, 2]
            b0, b1, b2, b3 = d[:, 3] / det, (-d[:, 1]) / det, (-d[:, 2]) / det, d[:, 0] / det
            tx, ty = x.astype(np.float64), y.astype(np.float64)
            m = np.stack([b0, b1, b2, b3, -(b0 * tx + b1 * ty), -(b2 * tx + b3 * ty)], 1).astype(F)
        ok = (det != 0.0) & np.isfinite(a).all(1) & np.isfinite(m).all(1)
        m[~ok] = np.nan
        r.update(m=m, nl=np.zeros(len(l), F))
    else:
        r.update(m=np.stack([a[:, 0], a[:, 1], x, a[:, 2], a[:, 3], y], 1).astype(F),
                 nl=_sq_norm64(a, np.stack([x, y], 1), prm.skip))
    return r


def cols(lafs2, H, prm):
    """frob_col of lafs2 [n,2,3] mapped through H^-1 -> dict (a [n,4], x, y, nt, s, tn)."""
    A, t = reproject(lafs2, inverse_h(H))
    A, s = frame_2x2(A, prm.up)
    x, y = t[:, 0].copy(), t[:, 1].copy()
    return dict(a=A, x=x, y=y, nt=x * x + y * y, s=s, tn=_sq_norm64(A, t, prm.skip))


def centre_dist(r, c):
    """centre_dist (gt_kernel's distance) [n1,n2]."""
    ax, ay = r["x"][:, None], r["y"][:, None]
    with np.errstate(all="ignore"):
        dot = fmaf32(ay, c["y"][None], ax * c["x"][None])
        return np.sqrt(np.abs(((c["nt"][None] + r["na"][:, None]) - F(2.0) * dot) + F(1e-12)))


def distances(r, c, prm, gated=True):
    """frob_scan's value for every (row, column) [n1,n2] fp32 (with the gate when prm.gate and gated)."""
    m = [r["m"][:, k][:, None] for k in range(6)]
    a = [c["a"][:, k][None] for k in range(4)]
    tx, ty = c["x"][None], c["y"][None]
    one = F(1.0)
    with np.errstate(all="ignore"):
        if prm.inv:
            m00, m01 = m[0] * a[0] + m[1] * a[2], m[0] * a[1] + m[1] * a[3]
            m10, m11 = m[2] * a[0] + m[3] * a[2], m[2] * a[1] + m[3] * a[3]
            e0, e3 = m00 - one, m11 - one
            d = ((e0 * e0 + m01 * m01) + m10 * m10) + e3 * e3
            if not prm.skip:
                r0 = (m[0] * tx + m[1] * ty) + m[4]
                r1 = (m[2] * tx + m[3] * ty) + m[5]
                d = d + (r0 * r0 + r1 * r1)
        else:
            if prm.skip:
                dot = ((m[0] * a[0] + m[1] * a[1]) + m[3] * a[2]) + m[4] * a[3]
            else:
                dot = (m[0] * a[0] + m[1] * a[1]) + m[2] * tx
                dot = (((dot + m[3] * a[2]) + m[4] * a[3]) + m[5] * ty) + one
            d = np.sqrt(np.abs(((c["tn"][None] + r["nl"][:, None]) - F(2.0) * dot) + F(1e-12)))
        if prm.gate and gated:
            far = (centre_dist(r, c) >= prm.cth).astype(F)
            if prm.coef > 0:
                ok = (np.abs(one - c["s"][None] / r["s1e"][:, None]) <= prm.coef).astype(F)
            else:
                ok = np.ones_like(d)
            d = ((one - ok) + far) * F(1000.0) + d
    return d.astype(F)


def reduce_rows(D, th):
    """The running (min, argmin) of frob_scan and the compaction -> (min_dist fp32, idx2 int64, true int64 ascending)."""
    n1, n2 = D.shape
    if n2 == 0:
        mn = np.full(n1, np.inf, F)
        return mn, np.zeros(n1, np.int64), np.zeros(0, np.int64)
    Dm = np.where(np.isnan(D), np.inf, D)
    lo = Dm.min(1)
    hit = (Dm == lo[:, None]) & (Dm < np.inf)
    has = hit.any(1)
    idx = np.where(has, hit.argmax(1), 0)
    mn = np.where(has, D[np.arange(n1), idx], np.inf).astype(F)
    return mn, idx.astype(np.int64), np.nonzero(mn <= F(th))[0].astype(np.int64)


def frobenius(lafs1, lafs2, H, prm):
    """One pair: every row of lafs1 [n1,2,3] against every row of lafs2 [n2,2,3] -> (min_dist, idx2, true)."""
    return reduce_rows(distances(rows(lafs1, prm), cols(lafs2, H, prm), prm), prm.th)


def frobenius_tent(lafs1, lafs2, tent, H, prm):
    """Tentative mode: rows lafs1[tent[:,0]] against columns lafs2[tent[:,1]]."""
    tent = np.asarray(tent, np.int64)
    return frobenius(np.asarray(lafs1)[tent[:, 0]], np.asarray(lafs2)[tent[:, 1]], H, prm)


# ---- agreement with the reference's fp32 values ----------------------------------------------------------------------------------------
def magnitudes(r, c, prm):
    """(M [n1,n2], kappa [n1]): M bounds the magnitude of the products summed into E = B A' - I and r = B (t' - t), entry by entry
    (|B| |A'| and |B| (|t'| + |t|), their largest entry plus 1); kappa is the condition number of row i's 2x2 part, which scales the
    error of either side's inverse."""
    with np.errstate(all="ignore"):
        B = np.abs(r["m"][:, :4].astype(np.float64))
        A = np.abs(c["a"].astype(np.float64))
        pa = [B[:, None, 0] * A[None, :, 0] + B[:, None, 1] * A[None, :, 2], B[:, None, 0] * A[None, :, 1] + B[:, None, 1] * A[None, :, 3],
              B[:, None, 2] * A[None, :, 0] + B[:, None, 3] * A[None, :, 2], B[:, None, 2] * A[None, :, 1] + B[:, None, 3] * A[None, :, 3]]
        M = np.max(np.stack(pa), 0) + 1.0
        if not prm.skip:
            tt = np.abs(c["x"].astype(np.float64))[None] + np.abs(r["x"].astype(np.float64))[:, None]
            tu = np.abs(c["y"].astype(np.float64))[None] + np.abs(r["y"].astype(np.float64))[:, None]
            M = np.maximum(M, np.maximum(B[:, None, 0] * tt + B[:, None, 1] * tu, B[:, None, 2] * tt + B[:, None, 3] * tu))
        Bi = r["m"][:, :4].astype(np.float64)
        fro = np.sqrt((Bi ** 2).sum(1))
        det = np.abs(Bi[:, 0] * Bi[:, 3] - Bi[:, 1] * Bi[:, 2])
        kappa = fro * fro / det                                         # |B|_F |B^-1|_F = |B|_F^2 / |det B| for 2x2
    return M, kappa


def d_bound(D, r, c, prm):
    """Per-element bound on |D_kernel - D_reference| (inv_to_eye): each of the 6 entries of E and r is within
    e = K_STEPS u kappa M of its exact value on either side, so |sqrt(D) - sqrt(D_ref)| <= 2 sqrt(6) e and
    |D - D_ref| <= 2 sqrt(6) e (2 sqrt(D) + 2 sqrt(6) e)."""
    M, kappa = magnitudes(r, c, prm)
    e = 2.0 * np.sqrt(6.0) * K_STEPS * U32 * kappa[:, None] * M
    return e * (2.0 * np.sqrt(np.abs(D.astype(np.float64))) + e)


def d_bound_expanded(D, r, c):
    """inv_to_eye = 0: the expanded distance's square is a difference of sums of at most 9 terms, each within K_STEPS u of the
    magnitudes |L1|^2 + |L2|^2, so |D - D_ref| <= K_STEPS u (|L1|^2 + |L2|^2) / max(D, sqrt(K_STEPS u (|L1|^2 + |L2|^2)))."""
    q = K_STEPS * U32 * (r["nl"].astype(np.float64)[:, None] + c["tn"].astype(np.float64)[None])
    return q / np.maximum(np.abs(D.astype(np.float64)), np.sqrt(q))
