"""An exact fp32 restatement of the scale-space kernels, operation by operation (test infrastructure, not product).

`blur_kernel` (pyramid.cu) and the bilinear sampler (`laf_sample_xy` + `bilinear_zero`,
common.cuh) are written with explicit fp32 roundings and fused multiply-adds in a fixed order, so their outputs are a function of
the inputs alone.  This module computes the same function on the CPU (or, for large images, on the device) from float64 tensor
operations: every fp32 step is one float64 operation whose exact result is then rounded to fp32, and the one step that float64
cannot do in one operation, the fused multiply-add, is `fmaf32` below.  No fp32 FMA is used anywhere, and separate float64 tensor
operations are never contracted, so a difference of one bit between a kernel and this module is a finding.

Next to it are float64 statements of the reference's own operations (the dense k x k blur with replicate padding, the closed-form
sampler), against which the kernels' fp32 error is bounded."""
import math

import numpy as np
import torch
import torch.nn.functional as F

import affnet_oracle as O

MAX_RADIUS = 12                     # blur_kernel<R> is instantiated for R = 1..12
U32 = 2.0 ** -24                    # unit roundoff of fp32


def _t64(x, device=None):
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(x)
    return x.to(device=device, dtype=torch.float64)


def fmaf32(a, b, c):
    """Correctly rounded fp32 fused multiply-add round(a*b + c) of fp32 values (tensors or arrays, broadcast), returned as fp32.

    The float64 product of two fp32 values is exact (48 significant bits).  TwoSum gives s + e == p + c exactly, s = fl64(p + c).
    Rounding s to fp32 rounds p + c correctly except when s lies exactly on an fp32 midpoint while e != 0: then the tie was
    broken without the tail, and the result moves to the neighbour on e's side."""
    is_np = isinstance(a, np.ndarray) or isinstance(b, np.ndarray) or isinstance(c, np.ndarray)
    dev = next((t.device for t in (a, b, c) if isinstance(t, torch.Tensor)), None)
    a, b, c = (_t64(v, dev) if isinstance(v, (torch.Tensor, np.ndarray)) else torch.tensor(float(v), dtype=torch.float64, device=dev)
               for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.to(torch.float32)
    r64 = r.to(torch.float64)
    below = r64 < s                                                   # s lies between r and its upper neighbour
    other = torch.where(below, torch.nextafter(r, torch.full_like(r, math.inf)), torch.nextafter(r, torch.full_like(r, -math.inf)))
    mid = (r64 != s) & ((r64 + other.to(torch.float64)) * 0.5 == s)
    fix = mid & (e != 0) & ((e > 0) == below)                         # the exact value lies beyond s, on the side of `other`
    r = torch.where(fix, other, r)
    return r.numpy() if is_np else r


def _f32(x):
    """Round float64 values to fp32 (one fp32 operation's rounding)."""
    return x.to(torch.float32)


# ---- blur ----------------------------------------------------------------------------------------------------------------
def taps(sigma):
    """make_taps (pyramid.cu): the 1-D factor of the reference's kernel with libm exp, normalised in float64, rounded to fp32."""
    k = O.gauss_kernel_size(sigma)
    half = k / 2.0
    step = (2.0 * half) / (k - 1) if k > 1 else 0.0
    e = [math.exp(-(x * x) / (2.0 * sigma * sigma)) for x in (half if i == k - 1 else -half + i * step for i in range(k))]
    s = 0.0
    for v in e:
        s += v
    return np.array([v / s for v in e], dtype=np.float64).astype(np.float32)


def radius(sigma):
    return O.gauss_kernel_size(sigma) // 2


def _pass(x, w, dim, descending=False):
    """acc = 0; acc = fmaf(w[k], x[clamp(i - R + k)], acc) for k = 0 .. 2R along `dim`: blur_kernel's order in either pass.
    `descending` sums k = 2R .. 0 instead (a deliberately wrong order, to show that the GPU tests see the difference)."""
    R = (len(w) - 1) // 2
    n = x.size(dim)
    idx = torch.arange(n, device=x.device)
    acc = torch.zeros_like(x, dtype=torch.float32)
    for k in (range(2 * R, -1, -1) if descending else range(2 * R + 1)):
        v = x.index_select(dim, (idx - R + k).clamp(0, n - 1))
        acc = fmaf32(torch.tensor(float(w[k]), dtype=torch.float32, device=x.device), v, acc)
    return acc


def blur32(x, sigma, descending=False):
    """blur_kernel's output for fp32 x [..., h, w]: horizontal pass over replicate-clamped columns, then vertical pass over
    replicate-clamped rows."""
    w = taps(sigma)
    x = x.to(torch.float32)
    return _pass(_pass(x, w, x.dim() - 1, descending), w, x.dim() - 2, descending)


def pyramid32(x, plan, descending=False):
    """ag_pyramid_build's levels for fp32 x [B, h, w] (or [h, w]) under an ag_pyramid_plan_t: pyr[o][l] as tensors of x's shape.

    Level 0 of octave 0 is the input when the plan's first blur sigma is 0 (init_sigma <= 0.5), otherwise its blur; level 0 of
    each later octave is [::2, ::2] of level n_levels - 2 of the previous one; level l > 0 is the blur of level l - 1."""
    x = x.to(torch.float32)
    pyr, cur = [], None
    for o in range(plan.n_octaves):
        if o == 0:
            bs = plan.blur_sigma[0][0]
            cur = blur32(x, bs, descending) if bs > 0.0 else x.clone()
        else:
            cur = pyr[o - 1][plan.n_levels - 2][..., ::2, ::2].contiguous()
        assert tuple(cur.shape[-2:]) == (plan.h[o], plan.w[o])
        levels = [cur]
        for l in range(1, plan.n_levels):
            cur = blur32(cur, plan.blur_sigma[o][l], descending)
            levels.append(cur)
        pyr.append(levels)
    return pyr


def blur64(x, sigma):
    """The reference's dense k x k cross-correlation with replicate padding (Utils.py:160-166), in float64, x [..., h, w]."""
    ker = torch.from_numpy(O.gauss_kernel_2d(sigma)).to(x.device)
    k = ker.shape[0]
    shp = x.shape
    x4 = x.to(torch.float64).reshape(-1, 1, shp[-2], shp[-1])
    y = F.conv2d(F.pad(x4, (k // 2,) * 4, "replicate"), ker.view(1, 1, k, k))
    return y.reshape(shp)


def pyramid64(x, plan):
    """The reference's pyramid (HandCraftedModules.py:23-56) in float64 under the same plan: a chain of dense blurs."""
    x = x.to(torch.float64)
    pyr = []
    for o in range(plan.n_octaves):
        if o == 0:
            bs = plan.blur_sigma[0][0]
            cur = blur64(x, bs) if bs > 0.0 else x.clone()
        else:
            cur = pyr[o - 1][plan.n_levels - 2][..., ::2, ::2].contiguous()
        levels = [cur]
        for l in range(1, plan.n_levels):
            cur = blur64(cur, plan.blur_sigma[o][l])
            levels.append(cur)
        pyr.append(levels)
    return pyr


def gamma(n):
    return n * U32 / (1.0 - n * U32)


def blur_bound(sigma):
    """Bound on |blur_kernel(x) - blur64(x)| / max|x| for one blur with k taps.

    Each pass is a k-term dot product with non-negative weights accumulated by FMAs: error <= gamma_k * sum(w) * max|x| (Higham 3.5),
    and the second pass adds its own gamma_k on values whose max norm is at most that of x.  The fp32 taps differ from the float64
    factor g by at most u * g each, so the separable kernel outer(w32, w32) differs from outer(g, g) by at most (2u + u^2) in l1
    norm.  The blur does not expand the max norm, so the bounds of a chain add (times its tiny growth sum(w32) <= 1 + k u)."""
    k = O.gauss_kernel_size(sigma)
    return (2.0 * gamma(k) + 2.0 * U32 + U32 * U32) * (1.0 + k * U32) ** 2


def pyramid_bounds(plan):
    """bound[o][l]: the sum of blur_bound over every blur on the chain from the input to level l of octave o (times max|x|)."""
    out, acc = [], 0.0
    for o in range(plan.n_octaves):
        row = []
        if o == 0:
            bs = plan.blur_sigma[0][0]
            acc = blur_bound(bs) if bs > 0.0 else 0.0
        else:
            acc = out[o - 1][plan.n_levels - 2]
        row.append(acc)
        for l in range(1, plan.n_levels):
            acc = acc + blur_bound(plan.blur_sigma[o][l])
            row.append(acc)
        out.append(row)
    return out


# ---- sampler -------------------------------------------------------------------------------------------------------------
def sample_xy32(lafs, h, w, PS, fma=None):
    """laf_sample_xy (common.cuh) for lafs fp32 [n, 2, 3]: fp32 (px, py) [n, PS, PS] with the kernel's roundings and FMAs."""
    fma = fma or fmaf32
    L = lafs.to(torch.float32).reshape(-1, 6)
    dev = L.device
    f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)   # noqa: E731
    ms, fw, fh = f32(float(min(h, w))), f32(float(w)), f32(float(h))
    mul = lambda a, b: _f32(_t64(a) * _t64(b))                           # noqa: E731  __fmul_rn
    sub = lambda a, b: _f32(_t64(a) - _t64(b))                           # noqa: E731  __fsub_rn
    a11, a12, tx = mul(L[:, 0], ms), mul(L[:, 1], ms), mul(L[:, 2], fw)
    a21, a22, ty = mul(L[:, 3], ms), mul(L[:, 4], ms), mul(L[:, 5], fh)
    inv_ps = _f32(torch.tensor(1.0, dtype=torch.float64) / float(np.float32(PS))).to(dev)   # 1.0f / (float)PS
    j = torch.arange(PS, dtype=torch.float32, device=dev)
    g = sub(mul(fma(f32(2.0), j, f32(1.0)), inv_ps), f32(1.0))          # x_j = y_j: (2j + 1) / PS - 1
    xj, yi = g.view(1, 1, PS), g.view(1, PS, 1)
    c = lambda v: v.view(-1, 1, 1)                                       # noqa: E731
    px = sub(fma(c(a11), xj, fma(c(a12), yi, c(tx))), f32(0.5))
    py = sub(fma(c(a21), xj, fma(c(a22), yi, c(ty))), f32(0.5))
    return px, py


def _taps4(img, px, py, sel=None):
    """The four zero-padded taps of bilinear_zero and the fractional parts, fp32.  img [m, h, w]; sel [n] picks img's plane per patch."""
    m, h, w = img.shape
    fx0, fy0 = torch.floor(px), torch.floor(py)
    # (int)floorf(): cvt.rzi.s32.f32 saturates to the int32 range; the int64 arithmetic below then never wraps
    x0 = fx0.to(torch.float64).clamp(-2.0 ** 31, 2.0 ** 31 - 1).to(torch.int64)
    y0 = fy0.to(torch.float64).clamp(-2.0 ** 31, 2.0 ** 31 - 1).to(torch.int64)
    ax, ay = _f32(_t64(px) - _t64(fx0)), _f32(_t64(py) - _t64(fy0))
    flat = img.reshape(m, h * w)
    plane = (torch.zeros(px.size(0), dtype=torch.int64, device=px.device) if sel is None else sel.to(px.device)).view(-1, 1, 1)

    def tap(yy, xx):
        ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        v = flat[plane.expand_as(yy), (yy.clamp(0, h - 1) * w + xx.clamp(0, w - 1))]
        return torch.where(ok, v, torch.zeros_like(v))

    return (tap(y0, x0), tap(y0, x0 + 1), tap(y0 + 1, x0), tap(y0 + 1, x0 + 1)), ax, ay


def sample32(img, lafs, PS, sel=None, fma=None):
    """ag_extract_patches for one channel: img fp32 [m, h, w] (m = 1, or one plane per patch with sel), lafs fp32 [n, 2, 3] ->
    [n, PS, PS] fp32, bit for bit: laf_sample_xy then bilinear_zero with __fmul_rn, __fmaf_rn, __fsub_rn and floorf."""
    fma = fma or fmaf32
    img = img.to(torch.float32)
    h, w = img.shape[-2:]
    px, py = sample_xy32(lafs, h, w, PS, fma)
    (v00, v01, v10, v11), ax, ay = _taps4(img, px, py, sel)
    one = torch.tensor(1.0, dtype=torch.float32, device=img.device)
    bx, by = _f32(_t64(one) - _t64(ax)), _f32(_t64(one) - _t64(ay))
    mul = lambda a, b: _f32(_t64(a) * _t64(b))   # noqa: E731
    top = fma(v01, ax, mul(v00, bx))
    bot = fma(v11, ax, mul(v10, bx))
    return fma(bot, ay, mul(top, by))


def sample64(img, lafs, PS):
    """The reference's sampler (affine_grid + grid_sample, bilinear, zeros, align_corners=False) in float64: img [1, h, w]."""
    h, w = img.shape[-2:]
    return O.extract_patches(img.reshape(1, 1, h, w), lafs.cpu(), PS, out_dtype=torch.float64)[:, 0]


def sample_bound(img, lafs):
    """Bound on |sample32 - sample64| over patches of img [h, w] at lafs [n, 2, 3] (PS-independent).

    The zero-padded bilinear interpolant is continuous and Lipschitz with constant G = the largest difference of two 4-adjacent
    pixels, the zero padding included, per unit of x plus the same per unit of y.  The fp32 sample point differs from the float64
    one by a few roundings of each term of A (x_j, y_i)^T + t: at most 8 u (|A| min(h, w) + |t| + 1) per coordinate, |A| the
    largest row sum of |A| and |t| the largest translation in pixels.  The fp32 combination of the four taps adds at most
    8 u max|I|."""
    h, w = img.shape[-2:]
    I = img.to(torch.float64).reshape(h, w)
    P = F.pad(I, (1, 1, 1, 1))
    G = max((P[:, 1:] - P[:, :-1]).abs().max().item(), (P[1:, :] - P[:-1, :]).abs().max().item())
    L = lafs.to(torch.float64).reshape(-1, 2, 3)
    A = (L[:, :, 0].abs() + L[:, :, 1].abs()).max().item() * min(h, w)
    t = max((L[:, 0, 2].abs() * w).max().item(), (L[:, 1, 2].abs() * h).max().item())
    return 2.0 * G * 8.0 * U32 * (A + t + 1.0) + 8.0 * U32 * I.abs().max().item()
