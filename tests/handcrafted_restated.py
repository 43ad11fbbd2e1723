"""An exact fp32 restatement of the hand-crafted estimators and the SIFT descriptor, operation by operation (test infrastructure, not
product).

`orientation_hist_warp` and `baumberg_warp` (handcrafted.cu) and `sift_block` (sift.cu) round every fp32 operation on its own, use fused
multiply-adds only where they are written as such, and reduce in a fixed order, so their outputs are a function of the patch alone.  This
module states the same function with numpy float32 arrays (numpy rounds each ufunc to fp32 and never fuses two of them) and `fmaf32` of
scale_space_restated.py for the written FMAs.  The device's `atan2f`, `cosf` and `sinf` cannot be restated; they are parameters: the GPU
tests pass the values of ag_debug_libm, the CPU tests correctly rounded float64 results (`atan2_cr` and friends below).

Arrays: patches [n,PS,PS] fp32, gk [PS,PS] fp32 (the window the kernel is handed), A / R [n,2,2], LAFs [n,2,3] normalised."""
import numpy as np

import geometry_restated as G
from scale_space_restated import fmaf32

F = np.float32
PI_F = F(np.pi)
TWO_PI_F = F(2.0 * np.pi)
U32 = 2.0 ** -24


def atan2_cr(y, x):
    """Correctly rounded atan2 of fp32 arrays (float64 result rounded to fp32; its error before rounding is far below half an fp32 ulp)."""
    with np.errstate(all="ignore"):
        return np.arctan2(np.asarray(y, np.float64), np.asarray(x, np.float64)).astype(np.float32)


def cos_cr(x):
    return np.cos(np.asarray(x, np.float64)).astype(np.float32)


def sin_cr(x):
    return np.sin(np.asarray(x, np.float64)).astype(np.float32)


def f32(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.float32))


def grad(P, wm, wp):
    """grad_at (common.cuh): gx = fl(fl(wm * x[j-1]) + fl(wp * x[j+1])) with replicate clamping, gy the same along rows."""
    P = f32(P)
    PS = P.shape[-1]
    idx = np.arange(PS)
    m, p = np.maximum(idx - 1, 0), np.minimum(idx + 1, PS - 1)
    wm, wp = F(wm), F(wp)
    with np.errstate(all="ignore"):
        gx = wm * P[:, :, m] + wp * P[:, :, p]
        gy = wm * P[:, m, :] + wp * P[:, p, :]
    return gx, gy


def _bin_index(bo0):
    """(int)bo0 of a floor value: cvt.rzi.s32.f32 turns NaN into 0."""
    return np.where(np.isnan(bo0), F(0), bo0).astype(np.int64)


# ---- the edge patches of tests/golden/handcrafted_edges.npz ------------------------------------------------------------------------
EDGE_NAMES = ("zero", "constant", "x_ramp", "y_ramp", "x_ramp_falling", "y_ramp_falling", "nan_pixel", "inf_pixel", "neg_inf_pixel",
              "neg_zero", "neg_zero_ramp", "huge", "v_shape", "checker")


def edge_patches(PS):
    """[len(EDGE_NAMES),PS,PS] fp32.  The falling x-ramp has gy = 0 and gx < 0 everywhere: atan2 = pi, o_big = 36, which fmod maps to
    bin 0 (and its SIFT angle lies on a bin boundary); the ramps give gradients exactly on bin boundaries.  `huge` holds values around
    1e19, so gx^2 + gy^2 overflows to inf.  `v_shape` is mirror-symmetric about the vertical axis: its two gradient directions fill
    bins 18 and 0 with the same weights, so the two smoothed bins tie up to the summation order."""
    i = np.arange(PS, dtype=np.float32).reshape(PS, 1) * np.ones((1, PS), np.float32)
    j = np.arange(PS, dtype=np.float32).reshape(1, PS) * np.ones((PS, 1), np.float32)
    rnd = np.random.default_rng(PS)
    base = np.floor(rnd.random((PS, PS)) * 256.0).astype(np.float32)
    out = {}
    out["zero"] = np.zeros((PS, PS), np.float32)
    out["constant"] = np.full((PS, PS), 97.0, np.float32)
    out["x_ramp"], out["y_ramp"] = 3.0 * j, 3.0 * i
    out["x_ramp_falling"], out["y_ramp_falling"] = 200.0 - 3.0 * j, 200.0 - 3.0 * i
    for name, v in (("nan_pixel", np.nan), ("inf_pixel", np.inf), ("neg_inf_pixel", -np.inf)):
        p = base.copy()
        p[PS // 2, (PS - 1) // 3] = v
        out[name] = p
    out["neg_zero"] = np.full((PS, PS), -0.0, np.float32)
    out["neg_zero_ramp"] = np.where(j < PS // 2, np.float32(-0.0), 2.0 * (j - PS // 2))
    out["huge"] = (base + 1.0) * np.float32(1e17)
    out["v_shape"] = np.abs(2.0 * j - (PS - 1))
    out["checker"] = 255.0 * ((i + j) % 2)
    return np.stack([out[n].astype(np.float32) for n in EDGE_NAMES])


# ---- orientation_hist_warp ------------------------------------------------------------------------------------------------------------
def orientation_weights(P, gk, atan2=atan2_cr):
    """Per pixel: the lower bin [n,NP] (int) and its weight (1 - frac) * mag [n,NP] fp32."""
    P = f32(P)
    n, PS = P.shape[0], P.shape[-1]
    gx, gy = grad(P, 0.5, -0.5)
    with np.errstate(all="ignore"):
        mag = np.sqrt((gx * gx + gy * gy) + F(1e-10)) * f32(gk)
        ori = f32(atan2(gy, gx))
        o_big = (F(36.0) * (ori + PI_F)) / TWO_PI_F
        bo0 = np.floor(o_big)
        wo1 = o_big - bo0
        bo0 = np.fmod(bo0, F(36.0))
        w = (F(1.0) - wo1) * mag
    return _bin_index(bo0).reshape(n, -1), w.reshape(n, -1)


def orientation_hist(P, gk, atan2=atan2_cr, order=None):
    """The kernel's histogram before smoothing, [n,36] fp32: bin b summed in raster order from +0 (lane b of the warp), / NP.
    `order` replaces the raster order by a permutation of the pixels (a deliberately wrong order, for the mutation checks)."""
    b, w = orientation_weights(P, gk, atan2)
    n, NP = w.shape
    acc = np.zeros((n, 36), np.float32)
    rows = np.arange(n)
    with np.errstate(all="ignore"):
        for i in (range(NP) if order is None else order):
            acc[rows, b[:, i]] = acc[rows, b[:, i]] + w[:, i]
        return acc / F(NP), ~np.isfinite(w).all(axis=1)


def smooth(h):
    """fmaf(0.33f, h[b+1], fmaf(0.34f, h[b], 0.33f * h[b-1])) with zero padding."""
    hp = np.zeros((h.shape[0], 38), np.float32)
    hp[:, 1:37] = h
    with np.errstate(all="ignore"):
        return fmaf32(F(0.33), hp[:, 2:38], fmaf32(F(0.34), hp[:, 1:37], F(0.33) * hp[:, 0:36]))


def bin_angle(idx):
    """-(fl(fl(2 pi_f * idx) / 36) - pi_f)."""
    return -((TWO_PI_F * np.asarray(idx).astype(np.float32)) / F(36.0) - PI_F)


def orientation_bins(P, gk, atan2=atan2_cr, order=None):
    """-> (smoothed bins [n,36], the winning bin [n]): the first maximum, or bin 0 when a weight is not finite."""
    h, bad = orientation_hist(P, gk, atan2, order)
    v = smooth(h)
    idx = np.where(bad, 0, np.argmax(np.where(np.isnan(v), -np.inf, v), axis=1))
    return v, idx


def orientation_angle(P, gk, atan2=atan2_cr, order=None):
    """ag_orientation_hist: the angle [n] fp32."""
    return bin_angle(orientation_bins(P, gk, atan2, order)[1])


def angle_to_R(ang, cos=cos_cr, sin=sin_cr):
    """angles2A as orientation_hist_pyr_kernel writes it: [[cos, sin], [-sin, cos]]."""
    c, s = f32(cos(ang)), f32(sin(ang))
    return np.stack([c, s, -s, c], axis=1).reshape(-1, 2, 2)


# ---- baumberg_warp --------------------------------------------------------------------------------------------------------------------
def _warp_sum(v):
    """warp_sum_f over the lane axis (last, 32): v += shfl_xor(v, o) for o = 16, 8, 4, 2, 1; every lane ends with lane 0's bits."""
    lanes = np.arange(32)
    with np.errstate(all="ignore"):
        for o in (16, 8, 4, 2, 1):
            v = v + v[..., lanes ^ o]
    return v[..., 0]


def lane_sums(t):
    """Per lane l the sum from +0 of t[i] over i = l, l + 32, ... in that order; t [n,NP] -> [n,32].  Padding with +0 changes nothing:
    the accumulator starts at +0 and so is never -0."""
    n, NP = t.shape
    K = -(-NP // 32)
    tp = np.zeros((n, K * 32), np.float32)
    tp[:, :NP] = t
    tp = tp.reshape(n, K, 32)
    acc = np.zeros((n, 32), np.float32)
    with np.errstate(all="ignore"):
        for k in range(K):
            acc = acc + tp[:, k]
    return acc


def _fl_ops(contract):
    """The two operations the contraction changes: x * y + z and x * y - z * w.  `contract` models nvcc fusing them (the earlier plain-C source)."""
    if not contract:
        return (lambda x, y, z: x * y + z), (lambda x, y, z: x * y - z)
    return (lambda x, y, z: fmaf32(x, y, z)), (lambda x, y, z: fmaf32(x, y, -z))


def baumberg_moments(P, gk, contract=False):
    """(a, b, c) [n] of the second-moment matrix: fl(fl(gx gx) g) etc., per-lane partial sums, the xor butterfly, / NP."""
    P = f32(P)
    n, NP = P.shape[0], P.shape[-1] * P.shape[-1]
    gx, gy = grad(P, -1.0, 1.0)
    g = f32(gk)
    out = []
    with np.errstate(all="ignore"):
        for u, v in ((gx, gx), (gx, gy), (gy, gy)):
            if contract:    # acc = fma(fl(u v), g, acc) per lane
                prod, t = (u * v).reshape(n, NP), np.broadcast_to(g, u.shape).reshape(n, NP)
                K = -(-NP // 32)
                acc = np.zeros((n, 32), np.float32)
                for k in range(K):
                    i = np.arange(32) + 32 * k
                    ok = i < NP
                    ii = np.minimum(i, NP - 1)
                    acc = np.where(ok, fmaf32(prod[:, ii], t[:, ii], acc), acc)
                s = acc
            else:
                s = lane_sums(((u * v) * g).reshape(n, NP))
            out.append(_warp_sum(s) / F(NP))
    return out


def inv_sqrt_rectify(a, b, c, contract=False):
    """invSqrt (HandCraftedModules.py:93-118) + abc2A + rectifyAffineTransformationUpIsUp (LAF.py:285-291), each torch operation one fp32
    operation in the expression's left-to-right order; A[0,1] = 0 * det.  -> A [n,2,2]."""
    fma_add, fma_sub = _fl_ops(contract)
    a, b, c = f32(a), f32(b), f32(c)
    with np.errstate(all="ignore"):
        eps = F(1e-12)
        mask = (b != 0).astype(np.float32)
        r1 = (mask * (c - a)) / fma_add(F(2.0), b, eps)
        sgn = np.where(r1 > 0, F(1), np.where(r1 < 0, F(-1), F(0)))          # torch.sign: 0 for NaN
        t1 = sgn / (np.abs(r1) + np.sqrt(fma_add(r1, r1, F(1.0))))
        r = F(1.0) / np.sqrt(fma_add(t1, t1, F(1.0)))
        t = t1 * r
        r = fma_add(r, mask, F(1.0) * (F(1.0) - mask))
        t = t * mask
        rr, tt, rt2 = r * r, t * t, (F(2.0) * r) * t
        x = F(1.0) / np.sqrt(fma_add(tt, c, fma_sub(rr, a, rt2 * b)) if contract else (rr * a - rt2 * b) + tt * c)
        z = F(1.0) / np.sqrt(fma_add(rr, c, fma_add(tt, a, rt2 * b)) if contract else (tt * a + rt2 * b) + rr * c)
        d = np.sqrt(x * z)
        x, z = x / d, z / d
        na = fma_add(rr, x, tt * z)
        nb = fma_add((-r) * t, x, (t * r) * z)
        nc = fma_add(tt, x, rr * z)
        a00, a01, a10, a11 = na, nb, nb, nc
        det = np.sqrt(np.abs(fma_sub(a00, a11, a10 * a01) + F(1e-10)))
        b2a2 = np.sqrt(fma_add(a01, a01, a00 * a00))
        A = np.stack([b2a2 / det, F(0.0) * det, fma_add(a11, a01, a10 * a00) / (b2a2 * det), det / b2a2], axis=1)
    return A.reshape(-1, 2, 2)


def baumberg(P, gk, contract=False):
    """ag_baumberg_shape: the up-is-up rectified A [n,2,2].  contract=True models nvcc contracting the earlier plain-C source."""
    a, b, c = baumberg_moments(P, gk, contract)
    return inv_sqrt_rectify(a, b, c, contract)


# ---- the pyramid variants -------------------------------------------------------------------------------------------------------------
def sample(img, lafs, PS):
    """extract_patches_pyr_kernel's sampler (laf_sample_xy + bilinear_zero) on one plane img [h,w] fp32: lafs [n,2,3] -> [n,PS,PS]."""
    import torch

    import scale_space_restated as R
    im = torch.from_numpy(f32(img)).reshape(1, *np.shape(img))
    return R.sample32(im, torch.from_numpy(f32(lafs)).reshape(-1, 2, 3), PS).numpy()


def orientation_hist_pyr(img, lafs, PS, gk, atan2=atan2_cr, cos=cos_cr, sin=sin_cr):
    """orientation_hist_pyr_kernel for keypoints sampled from one plane: R [n,2,2]."""
    return angle_to_R(orientation_angle(sample(img, lafs, PS), gk, atan2), cos, sin)


def baumberg_pyr(img, lafs, PS, gk, iters):
    """baumberg_pyr_kernel for keypoints sampled from one plane: sample at the working LAF, A = Baumberg step, base = A (first iteration)
    or mat2(A, base), working LAF = [base L0_A | t] before every further iteration.  -> base [n,2,2]."""
    L0 = f32(lafs).reshape(-1, 2, 3)
    cur, base = L0.copy(), None
    for it in range(iters):
        A = baumberg(sample(img, cur, PS), gk)
        base = A if it == 0 else G.mat2(A, base)
        if it != iters - 1:
            cur = G.left_multiply(base, L0)
    return base


# ---- sift_block -----------------------------------------------------------------------------------------------------------------------
def sift_geometry(PS):
    s = int(round(2.0 * (PS // 2) / 5.0))
    return 2 * s - 1, s


def _block_sum_128(v):
    """block_sum_128 over thread index t (last axis, 128): the xor butterfly within each warp of 32, then (w0 + w1) + (w2 + w3)."""
    n = v.shape[0]
    w = _warp_sum(v.reshape(n, 4, 32))
    with np.errstate(all="ignore"):
        return (w[:, 0] + w[:, 1]) + (w[:, 2] + w[:, 3])


def sift(P, gk, pk, clipval=0.2, atan2=atan2_cr, fused=True):
    """ag_sift_describe: [n,128] in [bin][cy][cx] order.  Thread t = bin + 8 cell pools angle bin t & 7 of cell t >> 3 with
    acc = fmaf(pk[dy,dx], v, acc) over dy, then dx; fused=False rounds the product first (the mutation check)."""
    P = f32(P)
    n, PS = P.shape[0], P.shape[-1]
    k, s = sift_geometry(PS)
    pk = f32(pk)
    gx, gy = grad(P, -1.0, 1.0)
    with np.errstate(all="ignore"):
        mag = np.sqrt((gx * gx + gy * gy) + F(1e-10)) * f32(gk)
        ori = f32(atan2(gy, gx + F(1e-8)))
        o_big = ((ori + TWO_PI_F) / TWO_PI_F) * F(8.0)
        bo0 = np.floor(o_big)
        wo1 = o_big - bo0
        b = _bin_index(bo0) & 7
        w0 = (F(1.0) - wo1) * mag
        w1 = wo1 * mag
        t = np.arange(128)
        tbin, cell = t & 7, t >> 3
        oy, ox = (cell >> 2) * s, (cell & 3) * s
        acc = np.zeros((n, 128), np.float32)
        for dy in range(k):
            for dx in range(k):
                bb, v0, v1 = b[:, oy + dy, ox + dx], w0[:, oy + dy, ox + dx], w1[:, oy + dy, ox + dx]
                v = np.where(bb == tbin, v0, np.where(((bb + 1) & 7) == tbin, v1, F(0)))
                acc = fmaf32(pk[dy, dx], v, acc) if fused else pk[dy, dx] * v + acc
        x = acc / np.sqrt(np.abs(_block_sum_128(acc * acc))[:, None] + F(1e-10))
        x = np.fmin(np.fmax(x, F(0)), F(clipval))                       # fmaxf / fminf: a NaN operand yields the other one
        x = x / np.sqrt(np.abs(_block_sum_128(x * x))[:, None] + F(1e-10))
        R = 3 * s + k                                                      # the pooled rows / columns
        bad = ~(np.isfinite(w0[:, :R, :R]) & np.isfinite(w1[:, :R, :R])).all(axis=(1, 2))
    out = np.empty((n, 128), np.float32)
    out[:, tbin * 16 + cell] = x
    out[bad] = np.nan
    return out
