"""An exact fp32 restatement of the detector's soft-argmax and keypoint write (affnet_b200/csrc/detect.cu), operation by operation
(test infrastructure, not product).

The soft-argmax of every candidate reads the 3x3x3 window of response maps around it (zero outside the image) and computes, in fp32,

    ns = sum sc_d r,  ny = sum (dy - 0.5) r,  nx = sum (dx - 0.5) r,  den = sum r,   (d, dy, dx in 0..2, sc_d = (float)sigma_d)

in one of two fixed orders:
- "taps" (detect_level_kernel, detect_fused_kernel): for d, dy, dx in turn, ns = fmaf(sc_d, r, ns), ny = fmaf(dy - 0.5, r, ny),
  nx = fmaf(dx - 0.5, r, nx), den = den + r;
- "rows" (detect_rows_kernel, detect_warp_kernel): per level and window row, hs = (l + c) + r and hx = fmaf(1.5, r, fmaf(0.5, c,
  -0.5 * l)); per level S = (hs0 + hs1) + hs2, ns = fmaf(sc_d, S, ns), ny += fmaf(1.5, hs2, fmaf(0.5, hs1, -0.5 * hs0)),
  nx += (hx0 + hx1) + hx2, den += S.
Both end in den + 1e-8f, sc = (ns / den) / min(h, w), y = ((ny / den) + y) / h, x = ((nx / den) + x) / w, and write_keypoint's
LAF row [a_scale * sc, +0, x; +0, a_scale * sc, y].

Every fp32 step here is one float64 tensor operation rounded to fp32 (float64 holds each fp32 sum, product and quotient closely
enough for that rounding to be the correctly rounded fp32 result, subnormal results included), and the fused steps are
`scale_space_restated.fmaf32`.  So a kernel that differs from these functions in one bit is wrong.  The functions run on the CPU or,
for large candidate sets, on the device; no library kernel is called.

Next to them is the float64 soft-argmax of the same fp32 inputs with a per-candidate bound that holds for any summation order, so
it covers both kernel orders, the oracle's F.conv2d and the reference's goldens alike.  The bound holds where every sum stays
finite in fp32 (`finite_sums`); where a sum overflows (images scaled far up), the fp32 functions are still exact IEEE arithmetic
(infinities and NaN pass through the float64 operations and `fmaf32` as through the kernel's), so the kernel's rows must have the
restatement's bits and NaN positions there (`same_bits`)."""
import numpy as np
import torch
import torch.nn.functional as F

import affnet_oracle as O
from scale_space_restated import fmaf32

U32 = 2.0 ** -24                         # unit roundoff of fp32
ETA = 2.0 ** -150                        # largest absolute rounding error of an fp32 result in the subnormal range
EPS_DEN = float(np.float32(1e-8))        # the 1e-8 added to den, an fp32 constant in both the kernels and the reference
K_ROUND = 32                             # roundings on any path from a tap to ns / ny / nx / den, in any order (27 adds + products)
N_OPS = 128                              # fp32 operations per sum, each with at most ETA of absolute error when its result is subnormal
ORDERS = ("taps", "rows")


def _d(x):
    return x.to(torch.float64)


def _f(x):
    """Round float64 values to fp32: one fp32 operation's rounding."""
    return x.to(torch.float32)


def add(a, b):
    return _f(_d(a) + _d(b))


def mul(a, b):
    return _f(_d(a) * _d(b))


def div(a, b):
    return _f(_d(a) / _d(b))


def level_maps(pyr_octave, sigmas, th=0.0):
    """The response maps of one octave, [n_levels, h, w] fp32: clamp(hessian_response - th, 0), the bits the kernels compute."""
    return torch.cat([torch.clamp(O.hessian_response(lv.reshape(1, 1, *lv.shape[-2:]).cpu(), s) - th, min=0)[0]
                      for lv, s in zip(pyr_octave, sigmas)])


def windows(maps3, pix):
    """The 3x3x3 zero-padded response windows [n, 3, 3, 3] (level, dy, dx) of pixels pix [n] (flat indices) of maps3 [3, h, w]."""
    _, h, w = maps3.shape
    P = F.pad(maps3, (1, 1, 1, 1))
    y, x = pix // w, pix % w
    dy = torch.arange(3, device=pix.device).view(1, 3, 1)
    dx = torch.arange(3, device=pix.device).view(1, 1, 3)
    flat = P.reshape(3, -1)
    idx = (y.view(-1, 1, 1) + dy) * (w + 2) + (x.view(-1, 1, 1) + dx)          # [n, 3, 3]
    return torch.stack([flat[d][idx] for d in range(3)], dim=1)


def sums32(R, sc, order, mutate=None):
    """(ns, ny, nx, den) fp32 [n] of windows R [n, 3, 3, 3] fp32 in the kernel order `order`; sc: the three fp32 scales.
    `mutate` names a deliberately wrong variant (tests only): "xy_swap" swaps the x and y offsets of the first window row."""
    n, dev = R.size(0), R.device
    z = torch.zeros(n, dtype=torch.float32, device=dev)
    ns, ny, nx, den = z, z, z, z
    f32 = lambda v: torch.tensor(float(v), dtype=torch.float32, device=dev)   # noqa: E731
    if order == "taps":
        for d in range(3):
            for dy in range(3):
                for dx in range(3):
                    r = R[:, d, dy, dx]
                    oy, ox = dy - 0.5, dx - 0.5
                    if mutate == "xy_swap" and dy == 0:
                        oy, ox = ox, oy
                    ns = fmaf32(f32(sc[d]), r, ns)
                    ny = fmaf32(f32(oy), r, ny)
                    nx = fmaf32(f32(ox), r, nx)
                    den = add(den, r)
        return ns, ny, nx, den
    assert order == "rows", order
    for d in range(3):
        hs, hx = [], []
        for j in range(3):
            l, c, r = R[:, d, j, 0], R[:, d, j, 1], R[:, d, j, 2]
            hs.append(add(add(l, c), r))
            if mutate == "xy_swap" and j == 0:      # the y offset (-0.5) in place of the x offsets of this row's sum
                hx.append(mul(f32(-0.5), hs[-1]))
            else:
                hx.append(fmaf32(f32(1.5), r, fmaf32(f32(0.5), c, mul(f32(-0.5), l))))
        S = add(add(hs[0], hs[1]), hs[2])
        ns = fmaf32(f32(sc[d]), S, ns)
        ny = add(ny, fmaf32(f32(1.5), hs[2], fmaf32(f32(0.5), hs[1], mul(f32(-0.5), hs[0]))))
        nx = add(nx, add(add(hx[0], hx[1]), hx[2]))
        den = add(den, S)
    return ns, ny, nx, den


def tail32(ns, ny, nx, den, pix, h, w, mutate=None):
    """The common tail: (sc, y, x) fp32 [n].  Mutations (tests only): "no_eps" (den without + 1e-8f), "den_times_min"
    (ns / (den * min_size)), "split_y" (ny / den / h + y / h)."""
    dev = ns.device
    f32 = lambda v: torch.tensor(float(v), dtype=torch.float32, device=dev)   # noqa: E731
    if mutate != "no_eps":
        den = add(den, f32(EPS_DEN))
    ms = f32(min(h, w))
    gy, gx = _f(pix // w), _f(pix % w)
    sc = div(ns, mul(den, ms)) if mutate == "den_times_min" else div(div(ns, den), ms)
    if mutate == "split_y":
        y = add(div(div(ny, den), f32(h)), div(gy, f32(h)))
    else:
        y = div(add(div(ny, den), gy), f32(h))
    x = div(add(div(nx, den), gx), f32(w))
    return sc, y, x


def lafs32(sc, y, x, a_scale=1.0):
    """write_keypoint: [n, 2, 3] fp32 rows [a_scale * sc, +0, x; +0, a_scale * sc, y]."""
    s = mul(torch.tensor(float(np.float32(a_scale)), dtype=torch.float32, device=sc.device), sc)
    z = torch.zeros_like(s)
    return torch.stack([s, z, x, z, s, y], dim=1).view(-1, 2, 3)


def softargmax32(maps3, sc, pix, order, a_scale=1.0, mutate=None):
    """The LAF rows [n, 2, 3] the kernel of `order` writes for pixels pix [n] of the detection level whose response maps (low,
    cur, high) are maps3 [3, h, w] fp32, scales sc (three floats).  Mutations (tests only): those of sums32 and tail32, and
    "scale_first" (a_scale applied to ns before the divisions)."""
    h, w = maps3.shape[-2:]
    R = windows(maps3, pix)
    ns, ny, nx, den = sums32(R, [float(np.float32(s)) for s in sc], order, mutate)
    if mutate == "scale_first":
        ns = mul(torch.tensor(float(np.float32(a_scale)), dtype=torch.float32, device=ns.device), ns)
    s, y, x = tail32(ns, ny, nx, den, pix, h, w, mutate)
    return lafs32(s, y, x, 1.0 if mutate == "scale_first" else a_scale)


# ---- float64 soft-argmax and its bound ------------------------------------------------------------------------------------------
def softargmax64(maps3, sc, pix, a_scale=1.0):
    """The exact soft-argmax of the same fp32 inputs, in float64, with a bound that holds for any summation order.

    Every tap reaches ns, ny, nx and den through at most K_ROUND roundings (the adds of any summation tree over 27 terms and the
    product, if not fused), each of relative error u or, with a subnormal result, absolute error ETA.  The terms of ns and den are
    nonnegative; those of ny and nx have weights |o| <= 1.5, so their error is relative to sum |o r|:
        |N^ - N| <= g (sum |o r|) + N_OPS ETA,   g = K u / (1 - K u);     den >= 1e-8 is normal, so |D^ - D| <= g D.
    The quotient then errs by (E_N + |N| g) / (D (1 - g)) plus its own rounding u |q| (+ ETA), the add of the pixel index by u |t|,
    and the final division by u |result| (+ ETA).  Returns (lafs64 [n, 2, 3], bound [n, 2, 3]), the bound zero on the exact-zero
    off-diagonals."""
    h, w = maps3.shape[-2:]
    R = _d(windows(maps3, pix)).reshape(-1, 3, 9)
    o = torch.tensor([-0.5, 0.5, 1.5], dtype=torch.float64, device=R.device)
    s64 = torch.tensor([float(np.float32(s)) for s in sc], dtype=torch.float64, device=R.device)
    oy = o.view(1, 1, 3, 1).expand(1, 3, 3, 3).reshape(1, 3, 9)
    ox = o.view(1, 1, 1, 3).expand(1, 3, 3, 3).reshape(1, 3, 9)
    Ns = (R * s64.view(1, 3, 1)).sum((1, 2))
    Ny, Nx = (R * oy).sum((1, 2)), (R * ox).sum((1, 2))
    Ay, Ax = (R * oy.abs()).sum((1, 2)), (R * ox.abs()).sum((1, 2))
    D = R.sum((1, 2)) + EPS_DEN
    g = K_ROUND * U32 / (1.0 - K_ROUND * U32)
    fudge = 2.0 ** -45                                              # float64 evaluation of the sums above
    gy, gx = _d(pix // w), _d(pix % w)
    ms = float(min(h, w))

    def quot(N, A):
        E = g * A + N_OPS * ETA + fudge * A
        q = N / D
        Eq = (E + N.abs() * g) / (D * (1.0 - g))
        return q, Eq + U32 * (q.abs() + Eq) + ETA

    qs, Es = quot(Ns, Ns)
    SC = qs / ms
    Esc = Es / ms + U32 * (SC.abs() + Es / ms) + ETA
    a = float(np.float32(a_scale))
    SCa = a * SC
    Esca = Esc if a == 1.0 else a * Esc + U32 * (SCa.abs() + a * Esc) + ETA

    def coord(N, A, gi, n):
        q, Eq = quot(N, A)
        t = q + gi
        Et = Eq + U32 * (t.abs() + Eq)
        v = t / n
        return v, Et / n + U32 * (v.abs() + Et / n) + ETA

    Y, Ey = coord(Ny, Ay, gy, float(h))
    X, Ex = coord(Nx, Ax, gx, float(w))
    z = torch.zeros_like(SC)
    lafs = torch.stack([SCa, z, X, z, SCa, Y], 1).view(-1, 2, 3)
    bound = torch.stack([Esca, z, Ex, z, Esca, Ey], 1).view(-1, 2, 3)
    return lafs, bound


def finite_sums(R):
    """Rows of windows R [n, 3, 3, 3] whose ns, ny, nx and den stay finite in fp32 in any summation order: the sum of the absolute
    terms (weights <= 1.5 and sc_d < 2^7), grown by every rounding on the way, is below FLT_MAX."""
    a = _d(R).abs().sum((1, 2, 3)) * 128.0 * (1.0 + 2.0 ** -18)
    return torch.isfinite(_d(R)).all(3).all(2).all(1) & (a < float(np.finfo(np.float32).max))


def same_bits(a, b):
    """fp32 tensors equal bit for bit where not NaN, and NaN at the same positions (NaN payloads differ between the CPU and the GPU)."""
    a, b = a.to(torch.float32).cpu(), b.to(torch.float32).cpu()
    if a.shape != b.shape:
        return False
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(bits(a)[~na], bits(b)[~nb])


def bound_ratio(lafs, ref64, bound):
    """max |lafs - ref64| / bound over the bounded entries (lafs fp32 [n, 2, 3]); the off-diagonals must be exactly +0."""
    if lafs.numel() == 0:
        return 0.0
    err = (_d(lafs).to(ref64.device) - ref64).abs()
    nz = bound > 0
    assert bool((err[~nz] == 0).all()), "off-diagonal LAF entries must be exactly zero"
    return float((err[nz] / bound[nz]).max())


# ---- candidate sets --------------------------------------------------------------------------------------------------------------
class Restated:
    """Restated LAF rows of the candidates seq [n] (slot << 27 | pixel) of a pyramid pyr[o][l] with scales sigmas[o][l] and
    threshold th: lafs32 in the kernel order `order` (None: not computed), and the float64 soft-argmax lafs64 with its bound.  The
    maps are the oracle's response maps of the pyramid; `device` runs the restatement there (the inputs are exact, so the bits do
    not depend on where it runs).  `maps` (per octave [n_levels, h, w]) replaces the Hessian maps, for response maps given directly.
    Rows of an OracleCandidates `c`: Restated(c.pyr, c.sigmas, c.seq, order, th=c.th)."""

    def __init__(self, pyr, sigmas, seq, order, a_scale=1.0, th=0.0, device=None, mutate=None, maps=None):
        from helpers import SEQ_PIX_BITS
        n_det = len(pyr[0]) - 2
        seq = torch.as_tensor(seq).to(torch.int64)
        self.lafs32 = torch.zeros(seq.numel(), 2, 3, dtype=torch.float32)
        self.lafs64 = torch.zeros(seq.numel(), 2, 3, dtype=torch.float64)
        self.bound = torch.zeros(seq.numel(), 2, 3, dtype=torch.float64)
        self.finite = torch.ones(seq.numel(), dtype=torch.bool)   # rows whose sums are finite in any order: the bound applies
        slot = seq >> SEQ_PIX_BITS
        pix = seq & ((1 << SEQ_PIX_BITS) - 1)
        for o in range(len(pyr)):
            if not bool(((slot >= o * n_det) & (slot < (o + 1) * n_det)).any()):
                continue
            m = maps[o] if maps is not None else level_maps(pyr[o], sigmas[o], th)
            m = m.to(device) if device is not None else m
            for k in range(n_det):
                sel = (slot == o * n_det + k).nonzero().view(-1)
                if sel.numel() == 0:
                    continue
                p = pix[sel].to(m.device)
                sc = sigmas[o][k:k + 3]
                if order is not None:
                    self.lafs32[sel] = softargmax32(m[k:k + 3], sc, p, order, a_scale, mutate).cpu()
                L64, B64 = softargmax64(m[k:k + 3], sc, p, a_scale)
                self.lafs64[sel], self.bound[sel] = L64.cpu(), B64.cpu()
                self.finite[sel] = finite_sums(windows(m[k:k + 3], p)).cpu()


def bits(x):
    """int32 view of fp32 values: -0 and +0 differ, every NaN payload is kept."""
    return x.contiguous().to(torch.float32).view(torch.int32)
