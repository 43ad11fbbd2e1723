"""An fp32 restatement of the keypoint geometry in the reference's operation order (test infrastructure, not product).

The reference computes the per-keypoint geometry with fp32 torch on the CPU: `torch.bmm` of 2x2 blocks (SparseImgRepresenter.py:136-137,
159-161, 175), batch_eig2x2 (Utils.py:168-175), checkTouchBoundary (LAF.py:98-104) and the coefficient products of
(de)normalizeLAFs (LAF.py:407-429).  A 2x2 product there rounds both products and then adds them, fl(fl(a*b) + fl(c*d)) (from an
accumulator of +0), and a boundary corner is summed as fl(fl(fl(h0*x) + fl(h1*y)) + h2).  This module states each step as one numpy float32 operation: numpy
rounds every ufunc to fp32 and never fuses two of them, so the results are a function of the inputs alone, and the kernels of
geometry.cu (with mat2_mul / laf_left_mul of common.cuh) must reproduce them bit for bit.

Arrays are float32 numpy: A [n,2,2], LAFs [n,2,3], R [n,2,2]."""
import numpy as np

F = np.float32
SIXTH = F(1.0 / 6.0)                # `ratio > (1./6.)` compares an fp32 tensor with the scalar rounded to fp32
EPS_L2 = F(1e-8)                    # l2 + 1e-8 (SparseImgRepresenter.py:148)
CORNERS = ((-1, -1), (-1, 1), (1, -1), (1, 1))   # the columns of checkTouchBoundary's pts


def f32(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.float32))


def dot2(a, b, c, d):
    """fl(fl(0 + fl(a*b)) + fl(c*d)): one entry of a 2x2 torch.bmm, whose accumulator starts at +0 (the same as fl(fl(a*b) + fl(c*d))
    except that two -0 products sum to +0)."""
    return (F(0) + a * b) + c * d


def mat2(A, B):
    """A @ B for [n,2,2] (base_A <- bmm(A, base_A), SparseImgRepresenter.py:136)."""
    A, B = f32(A), f32(B)
    out = np.empty(np.broadcast_shapes(A.shape, B.shape), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(2):
            for j in range(2):
                out[:, i, j] = dot2(A[:, i, 0], B[:, 0, j], A[:, i, 1], B[:, 1, j])
    return out


def compose(A, L):
    """[bmm(A, L[:, :, :2]) | L[:, :, 2]] (SparseImgRepresenter.py:137, 161); also the working LAF of the next shape iteration."""
    A, L = f32(A), f32(L)
    out = L.copy()
    out[:, :, :2] = mat2(A, L[:, :, :2])
    return out


left_multiply = compose


def rotate(L, R):
    """[bmm(L[:, :, :2], R) | L[:, :, 2]] (SparseImgRepresenter.py:175)."""
    L, R = f32(L), f32(R)
    out = L.copy()
    out[:, :, :2] = mat2(L[:, :, :2], R)
    return out


def scale(L, ac, xc, yc):
    """coef * LAFs with coef = [[ac, ac, xc], [ac, ac, yc]] (LAF.py:412-417, 424-429): one fp32 product per entry."""
    coef = np.array([[ac, ac, xc], [ac, ac, yc]], np.float32)
    return f32(L) * coef


def denorm_coefs(w, h):
    """denormalizeLAFs(w, h): min(h, w), w, h as fp32."""
    return F(min(float(h), float(w))), F(float(w)), F(float(h))


def norm_coefs(w, h):
    """normalizeLAFs(w, h): ones(..).float() / min(h, w) divides in fp32; 1.0 / w and 1.0 / h are Python doubles stored into the fp32
    coefficient tensor (pipeline.cu and LAF.normalizeLAFs build the same three numbers)."""
    return F(1.0) / F(min(float(h), float(w))), F(1.0 / float(w)), F(1.0 / float(h))


def batch_eig2x2(A):
    """Utils.py:168-175, every torch op as one fp32 op (l1 and l2 keep the reference's mask arithmetic, so a rejected row whose
    trace + delta is not finite gives NaN there, as in the reference).  -> (l1, l2)."""
    A = f32(A)
    a00, a01, a10, a11 = A[:, 0, 0], A[:, 0, 1], A[:, 1, 0], A[:, 1, 1]
    with np.errstate(invalid="ignore", over="ignore"):
        trace = a00 + a11
        delta1 = trace * trace - F(4) * (a00 * a11 - a10 * a01)
        mask = (delta1 > 0).astype(np.float32)
        delta = np.sqrt(np.abs(delta1))
        l1 = mask * (trace + delta) / F(2) + F(1000.0) * (F(1) - mask)
        l2 = mask * (trace - delta) / F(2) + F(0.0001) * (F(1) - mask)
    return l1, l2


def eig_ratio(A):
    """|l1 / (l2 + 1e-8)| (SparseImgRepresenter.py:148)."""
    l1, l2 = batch_eig2x2(A)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return np.abs(l1 / (l2 + EPS_L2))


def eig_ok(A):
    """(ratio < 6) & (ratio > fp32(1/6)) (SparseImgRepresenter.py:149)."""
    r = eig_ratio(A)
    return (r < F(6.0)) & (r > SIXTH)


def corners(NL):
    """The four corners of checkTouchBoundary, ((0 + h0*x) + h1*y) + h2 per row, as torch.matmul sums them: -> [n,2,4]."""
    NL = f32(NL)
    out = np.empty((NL.shape[0], 2, 4), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for c, (x, y) in enumerate(CORNERS):
            out[:, :, c] = ((F(0) + NL[:, :, 0] * F(x)) + NL[:, :, 1] * F(y)) + NL[:, :, 2]
    return out


def touch_ok(NL):
    """~checkTouchBoundary's rejection: no corner coordinate > 1 or < 0 (NaN corners pass, as in the reference)."""
    c = corners(NL)
    with np.errstate(invalid="ignore"):
        return ~((c > 1) | (c < 0)).any(axis=(1, 2))


def shape_mask(A, L):
    """The keep mask of getAffineShape (SparseImgRepresenter.py:147-149) for base_A = A and detector LAFs L."""
    return eig_ok(A) & touch_ok(compose(A, L))


def select(mask, resp, num_features, out_cap):
    """The filter's selection (include/affnet_b200.h): if the survivors S exceed num_features > 0, the top num_features of
    resp * mask by value, descending, ties to the lowest row (-0 equals +0); else all survivors in row order.  The first out_cap rows
    of that answer are returned.  -> (rows, values): values are resp * mask at those rows in the sorted case (a rejected row that
    makes the cut is returned with the reference's zero), resp otherwise."""
    resp = f32(resp)
    S = int(mask.sum())
    if num_features > 0 and S > num_features:
        key = resp * mask.astype(np.float32)
        rows = np.lexsort((np.arange(len(key)), -key.astype(np.float64)))[:num_features][:out_cap]
        return rows, key[rows]
    rows = np.nonzero(mask)[0][:out_cap]
    return rows, resp[rows]


def shape_filter(A, resp, L, num_features, out_cap=None):
    """getAffineShape's tail for one image: -> (rows, resp_out [m], lafs_out [m,2,3])."""
    mask = shape_mask(A, L)
    rows, vals = select(mask, resp, num_features, len(mask) if out_cap is None else out_cap)
    return rows, vals, compose(f32(A)[rows], f32(L)[rows])


# ---- LAFs2ellT (LAF.py:35-51, bsvd2x2 :106-144) in float64: what the device's fp32 ellipses are bounded against ------------------------
def lafs_to_ell64(L):
    """[n,2,3] -> [n,5] float64 by the reference's closed form (only U and the singular values enter the result)."""
    L = np.asarray(L, np.float64)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        scale = np.sqrt(L[:, 0, 0] * L[:, 1, 1] - L[:, 0, 1] * L[:, 1, 0] + 1e-10)
        a = L[:, :, :2] / scale[:, None, None]
        s00 = a[:, 0, 0] ** 2 + a[:, 0, 1] ** 2
        s01 = a[:, 0, 0] * a[:, 1, 0] + a[:, 0, 1] * a[:, 1, 1]
        s11 = a[:, 1, 0] ** 2 + a[:, 1, 1] ** 2
        phi = 0.5 * np.arctan2(2 * s01 + 1e-12, s00 - s11 + 1e-12)
        c, s = np.cos(phi), np.sin(phi)
        dif = np.sqrt((s00 - s11) ** 2 + 4 * s01 * s01 + 1e-12)
        sig0, sig1 = np.sqrt((s00 + s11 + dif) / 2), np.sqrt((s00 + s11 - dif) / 2)
        w0, w1 = 1 / (scale * scale * sig0 * sig0), 1 / (scale * scale * sig1 * sig1)
        out = np.stack([L[:, 0, 2], L[:, 1, 2], c * w0 * c + s * w1 * s, c * w0 * s - s * w1 * c, s * w0 * s + c * w1 * c], 1)
    return out
