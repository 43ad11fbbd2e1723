"""The numerics of the second-generation tensor-core net engine (ENGINE_TC2 / ENGINE_TC2_BF16, tcx_first.cuh / tcx_conv.cuh / tc_head.cuh)
restated in float64, with a per-element error bound (test infrastructure, not product).

What is exact here:
- BatchNorm folding and the power-of-two weight scales, in fp32 as ag_net_create computes them (`fold`, `pow2_scale`);
- the operands the tensor cores multiply: weights as fp16 (bf16) `hi` [+ `lo` = round(v - hi)] of the scaled folded weights, where
  `tcx_split_w` keeps a residual; activations as the decoded planes (`hi + lo` for AffNet / OriNet, one plane for HardNet);
- the first kernel's input normalisation, restated bit for bit in fp32 (`input_norm32`) and split into its `hi + lo` planes.
A layer's float64 value is the exact convolution of those operands.  What the engine rounds is bounded per element (`conv_layer`):
- the operand products it leaves out (A_lo * W_lo);
- fp32 tensor-core accumulation.  Model: every wgmma K = 16 step aligns its 16 products and the incoming accumulator c_t to the largest
  of them and truncates, so it is off by at most C_ACC * 2^-23 * (|c_t| + sum |a b|); c_t is taken from the float64 partial sums in the
  kernel's issue order (kernel row dy, then 16 input channels, then the hi*hi, hi*lo, lo*hi MMAs);
- the epilogue's two fp32 adds of the three taps and fmaf(acc, 1/scale, bias);
- the store: 2^-22 |y| + the fp16 subnormal step for `hi + lo` planes.  A single fp16 / bf16 plane is not bounded but checked as
  "admissible": the stored value must be round-to-nearest of some value within the bound (`admissible`).
The heads are restated the same way (`affori_head`, `hardnet_head`); tanhf is allowed its CUDA Programming Guide bound of 2 ulp.

Tensors are float64 on any device; patches [n,1,32,32]; activations [n,C,H,H]; conv weights [co,ci,3,3]."""
import math

import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -24          # fp32 unit roundoff
C_ACC = 4.0             # accumulation model constant: 17 aligned terms truncated with 3 guard bits (17 / 8) plus the final truncation,
                        # rounded up; the GPU tests print the measured error / bound ratio
MARGIN = 1.0 + 2.0 ** -9
FMT = {"fp16": (11, -14), "bf16": (8, -126), "fp32": (24, -126)}    # significand bits, smallest normal exponent
AFF_CFG = [(1, 16, 1), (16, 16, 1), (16, 32, 2), (32, 32, 1), (32, 64, 2), (64, 64, 1)]
HARD_CFG = [(1, 32, 1), (32, 32, 1), (32, 64, 2), (64, 64, 1), (64, 128, 2), (128, 128, 1)]
CONV_IDX = [0, 3, 6, 9, 12, 15]
F32 = np.float32


def cfg_of(kind):
    return HARD_CFG if kind == "hardnet" else AFF_CFG


# ---- rounding ------------------------------------------------------------------------------------------------------------------
def _exp_q(x, fmt):
    p, emin = FMT[fmt]
    _, e = torch.frexp(x)                       # x = m 2^e, 0.5 <= |m| < 1
    return torch.clamp(e.to(torch.int64) - p, min=emin - p + 1)


def rnd(x, fmt):
    """Round-to-nearest-even of float64 values to fp16 / bf16 / fp32 (subnormals included; no overflow handling)."""
    x = x.to(torch.float64)
    q = _exp_q(x, fmt)
    return torch.ldexp(torch.round(torch.ldexp(x, -q)), q)


def rnd_rz(x, fmt):
    """Round toward zero (a mutation of the stores in the CPU sensitivity tests)."""
    x = x.to(torch.float64)
    q = _exp_q(x, fmt)
    return torch.ldexp(torch.trunc(torch.ldexp(x, -q)), q)


def ulp(x, fmt):
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), _exp_q(x.to(torch.float64), fmt))


def split(v, fmt, lo=True):
    """hi = round(v), lo = round(v - hi) (v - hi is exact in fp32 for fp32 v): the engine's split_pack / tcx_pack_layer."""
    hi = rnd(v, fmt)
    return hi, (rnd(v - hi, fmt) if lo else torch.zeros_like(hi))


# ---- weights as ag_net_create folds and packs them ------------------------------------------------------------------------------
def pow2_scale(w):
    """nets_simt.cu pow2_scale: the power of two that brings max |w| near 2^13."""
    wmax = float(np.max(np.abs(w))) if np.size(w) else 0.0
    if wmax <= 0.0:
        return 1.0
    return math.ldexp(1.0, 13 - math.frexp(wmax)[1])


def fold(sd, kind):
    """BatchNorm folded in fp32 (ag_net_create): W * (1 / sqrtf(var + 1e-5)), -mean * invstd.  -> [(W fp32 [co,ci,3,3], b fp32 [co])] * 6
    and the head: AffNet / OriNet (w [no,c,8,8], bias [no]); HardNet (w [128,128,8,8], bn scale [128], bn shift [128])."""
    g = lambda k: np.asarray(sd[k].detach().cpu().numpy() if torch.is_tensor(sd[k]) else sd[k], F32)
    layers = []
    for i in CONV_IDX:
        w, m, v = g("features.%d.weight" % i), g("features.%d.running_mean" % (i + 1)), g("features.%d.running_var" % (i + 1))
        inv = F32(1.0) / np.sqrt(v + F32(1e-5))
        layers.append((w * inv[:, None, None, None], (-m) * inv))
    if kind == "hardnet":
        m, v = g("features.20.running_mean"), g("features.20.running_var")
        s = np.sqrt(v + F32(1e-5))
        head = (g("features.19.weight"), F32(1.0) / s, (-m) / s)
    else:
        head = (g("features.19.weight"), g("features.19.bias"))
    return layers, head


def split_w(kind, layer, sw2=1, sw3=1):
    """tcx_split_w: whether layer `layer` (1..6) keeps a weight residual (AffNet / OriNet always; HardNet layers 2-3)."""
    if kind != "hardnet":
        return 1
    return {2: sw2, 3: sw3}.get(layer, 0) if layer >= 2 else 1


def operands(kind, sd, fmt="fp16", sw2=1, sw3=1):
    """The engine's weight operands, unscaled, as float64: per layer (w_hi, w_lo) with w = (hi + lo) / scale, the fp32 bias, and the head's
    operands.  Layer 1's weights always carry a residual (tcx_first.cuh)."""
    layers, head = fold(sd, kind)
    out = []
    for l, (w, b) in enumerate(layers, 1):
        s = pow2_scale(w)
        hi, lo = split(torch.from_numpy(w).double() * s, fmt, lo=bool(split_w(kind, l, sw2, sw3)))
        out.append((hi / s, lo / s, torch.from_numpy(b).double()))
    if kind == "hardnet":
        hw, bs, bsh = head     # fp16: times a power of two, its inverse folded into the BatchNorm scale; bf16: as they are
        s = pow2_scale(hw) if fmt == "fp16" else 1.0
        hh = (rnd(torch.from_numpy(hw).double() * s, fmt) / s, torch.zeros(1, dtype=torch.float64), torch.from_numpy(bs).double(), torch.from_numpy(bsh).double())
    else:
        hw, hb = head
        s = pow2_scale(hw)
        hi, lo = split(torch.from_numpy(hw).double() * s, "fp16")
        hh = (hi / s, lo / s, torch.from_numpy(hb).double())
    return out, hh


# ---- input normalisation, bit for bit (tcx_first.cuh producers) -----------------------------------------------------------------
def _butterfly(a, add=None):
    """xor-shuffle sum over the last axis (32 lanes), as every lane sees it after offsets 16, 8, 4, 2, 1.  add(x, y): the fp32 sum (default
    the arrays' own +, for fp32 arrays)."""
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        a = a + a[..., idx ^ o] if add is None else add(a, a[..., idx ^ o])
    return a[..., 0]


def _fmaf(a, b, c):
    from scale_space_restated import fmaf32
    return fmaf32(np.asarray(a, F32), np.asarray(b, F32), np.asarray(c, F32))


def input_norm32(P):
    """(v - mean) * (1 / (sqrtf(q / 1023) + 1e-7)) with tcx_first.cuh's fp32 sums: thread (warp pw, lane) holds pixels
    (4 pw + lane / 8, 8 k + lane % 8), k = 0..3.  -> fp32 numpy [n,32,32]."""
    P = np.asarray(P, F32).reshape(-1, 32, 32)
    n = P.shape[0]
    pw, lane, k = np.meshgrid(np.arange(8), np.arange(32), np.arange(4), indexing="ij")
    v = P[:, 4 * pw + lane // 8, 8 * k + lane % 8]                        # [n, 8 warps, 32 lanes, 4]
    sm = (v[..., 0] + v[..., 1]) + (v[..., 2] + v[..., 3])
    red = _butterfly(sm)                                                   # [n, 8]
    mean = (((red[:, 0] + red[:, 1]) + (red[:, 2] + red[:, 3])) + ((red[:, 4] + red[:, 5]) + (red[:, 6] + red[:, 7]))) / F32(1024)
    d = v - mean[:, None, None, None]
    qs = np.zeros(d.shape[:3], F32)
    for kk in range(4):
        qs = _fmaf(d[..., kk], d[..., kk], qs)
    rq = _butterfly(qs)
    tot = ((rq[:, 0] + rq[:, 1]) + (rq[:, 2] + rq[:, 3])) + ((rq[:, 4] + rq[:, 5]) + (rq[:, 6] + rq[:, 7]))
    inv = F32(1) / (np.sqrt(tot / F32(1023)) + F32(1e-7))
    return ((P - mean[:, None, None]) * inv[:, None, None]).astype(F32)


# ---- layers -------------------------------------------------------------------------------------------------------------------
def _taps(x, dy, dx, stride, Ho):
    return x[:, :, dy: dy + stride * Ho: stride, dx: dx + stride * Ho: stride]


def conv_layer(x, w_hi, w_lo, bias, stride, xr=None, a_lo=None, first=False):
    """One conv + folded BN layer on the exact operands: y = conv(x, w_hi + w_lo) + bias (before the ReLU) and the bound B on
    |computed - y| before the store.  x: the input (the sum of its planes), xr: a radius the true input may lie within (None: exact),
    a_lo: |activation residual| when the input has a lo plane (its lo * w_lo products are left out).  first: layer 1 (one K = 16 step per
    pixel, no x shifts)."""
    w = w_hi + w_lo
    m = 1 + int(bool(w_lo.abs().max() > 0)) + int(a_lo is not None or first)
    ax = x.abs() if xr is None else x.abs() + xr
    if first:
        y = F.conv2d(x, w, padding=1)
        P = F.conv2d(ax, w.abs(), padding=1)
        B = C_ACC * 2.0 ** -23 * 3 * P * MARGIN + U * P                   # hi*hi, lo*hi, hi*lo in one step; AffNet adds two columns
    else:
        n, ci, H, _ = x.shape
        Ho = H // stride
        xp, ap = F.pad(x, (1, 1, 1, 1)), F.pad(ax, (1, 1, 1, 1))
        y = 0.0
        acc_b = 0.0
        tap_abs = 0.0
        for dx in range(3):
            S = torch.zeros(n, w.shape[0], Ho, Ho, dtype=torch.float64, device=x.device)
            ab = torch.zeros_like(S)
            for dy in range(3):
                xs, as_ = _taps(xp, dy, dx, stride, Ho), _taps(ap, dy, dx, stride, Ho)
                for j in range(ci // 16):
                    sl = slice(16 * j, 16 * j + 16)
                    Pg = torch.einsum("nchw,oc->nohw", as_[:, sl], w[:, sl, dy, dx].abs())
                    ab += m * (S.abs() + Pg)
                    S = S + torch.einsum("nchw,oc->nohw", xs[:, sl], w[:, sl, dy, dx])
            y = y + S
            acc_b = acc_b + C_ACC * 2.0 ** -23 * ab * MARGIN
            tap_abs = tap_abs + S.abs() + C_ACC * 2.0 ** -23 * ab * MARGIN
        B = acc_b + 2.0001 * U * tap_abs                                  # two fp32 adds of the three taps
    if xr is not None:
        B = B + F.conv2d(xr, w.abs(), stride=stride, padding=1)
    if a_lo is not None:
        B = B + F.conv2d(a_lo, w_lo.abs(), stride=stride, padding=1)
    y = y + bias.view(1, -1, 1, 1)
    B = B + U * (y.abs() + B)                                             # fmaf(acc, 1/scale, bias)
    return y, B


def pair_store_bound(y, B):
    """hi + lo fp16 planes of relu(y): |stored - relu(y)| <= this."""
    return B + 2.0 ** -22 * (y.abs() + B) + 2.0 ** -24


def admissible(y, B, fmt):
    """[lo, hi]: the values round-to-nearest can store for relu(t), |t - y| <= B."""
    return rnd(torch.clamp(y - B, min=0), fmt), rnd(torch.clamp(y + B, min=0), fmt)


def store_interval(y, B, fmt, pair):
    """The interval the stored layer output lies in, as (centre, radius): for a layer that is not observed (layer 1)."""
    if pair:
        return torch.clamp(y, min=0), pair_store_bound(y, B)
    lo, hi = admissible(y, B, fmt)
    return 0.5 * (lo + hi), 0.5 * (hi - lo)


def a_lo_of(x, fmt="fp16"):
    """|x - round(x)|: the size of the lo plane of a decoded hi + lo activation (the same at a tie whichever way hi went)."""
    return (x - rnd(x, fmt)).abs()


# ---- layer 1 from the patch ----------------------------------------------------------------------------------------------------
def layer1(P, w_hi, w_lo, bias, fmt, device=None):
    """Layer 1 of the first kernel from the patches: the input planes hi + lo of input_norm32 in `fmt`, both weight parts."""
    xn = torch.from_numpy(input_norm32(np.asarray(P.cpu() if torch.is_tensor(P) else P))).double().to(device).unsqueeze(1)
    a_hi, a_lo = split(xn, fmt)
    y, B = conv_layer(a_hi + a_lo, w_hi.to(device), w_lo.to(device), bias.to(device), 1, first=True)
    B = B + F.conv2d(a_lo.abs(), w_lo.abs().to(device), padding=1)        # lo * lo left out
    return y, B


# ---- heads --------------------------------------------------------------------------------------------------------------------
def _spacing32(t):
    return torch.clamp(ulp(t, "fp32"), min=2.0 ** -149)


def affori_head(feat, w_hi, w_lo, bias, kind):
    """tc_headx_kernel on the layer-6 features feat [n,64,8,8] (hi + lo): the pre-tanh values z [n,no] and their bound, and the raw
    outputs (AffNet: 1 + tanh, tanh, 1 + tanh; OriNet: the mean of the nine tanh of each map) with their bound (tanhf within 2 ulp).
    The GEMM runs pixel by pixel (64 channels per K stage, fresh accumulator per stage, the stage sums added in fp32)."""
    n = feat.shape[0]
    w = w_hi + w_lo
    if kind == "orinet":                       # the padded 8x8 conv on the 8x8 map: 18 dot products against shifted kernels
        wp = F.pad(w, (1, 1, 1, 1))            # [2,64,10,10]
        weff = torch.stack([wp[ch, :, 2 - oy: 10 - oy, 2 - ox: 10 - ox] for ch in range(2) for oy in range(3) for ox in range(3)])
        wl = F.pad(w_lo, (1, 1, 1, 1))
        weff_lo = torch.stack([wl[ch, :, 2 - oy: 10 - oy, 2 - ox: 10 - ox] for ch in range(2) for oy in range(3) for ox in range(3)])
        bias_e = bias.repeat_interleave(9)
    else:
        weff, weff_lo, bias_e = w, w_lo, bias
    fk = feat.reshape(n, 64, 64).transpose(1, 2)                           # [n, pixel, c]
    wk = weff.reshape(-1, 64, 64).transpose(1, 2)                          # [o, pixel, c]
    prod = torch.einsum("npc,opc->nopc", fk, wk).reshape(n, -1, 64, 4, 16)
    G = prod.sum(-1)                                                       # [n,o,pixel,group]
    Pg = prod.abs().sum(-1)
    Sprev = G.cumsum(-1) - G
    stage_b = C_ACC * 2.0 ** -23 * 3 * (Sprev.abs() + Pg).sum(-1) * MARGIN  # [n,o,pixel]
    T = G.sum(-1).cumsum(-1)                                               # running fp32 totals over the stages
    acc = T[..., -1]
    # the stage sums of the hi columns and of the A_hi * W_lo columns are added up separately, then added (the lo totals stay below
    # 2^-10 of the running sums of |products|)
    Bacc = stage_b.sum(-1) + U * (T.abs().sum(-1) + 2.0 ** -10 * Pg.sum(-1).cumsum(-1).sum(-1)) + U * (acc.abs() + stage_b.sum(-1))
    a_lo = a_lo_of(feat).reshape(n, 64, 64).transpose(1, 2)
    Bacc = Bacc + torch.einsum("npc,opc->no", a_lo, weff_lo.reshape(-1, 64, 64).transpose(1, 2).abs())
    z = acc + bias_e
    Bz = Bacc + U * (z.abs() + Bacc)
    t = torch.tanh(z)
    Bt = Bz + 2 * _spacing32(t)
    if kind == "affnet":
        raw = torch.stack([1 + t[:, 0], t[:, 1], 1 + t[:, 2]], 1)
        Braw = Bt + U * (raw.abs() + Bt)
        return z, Bz, raw, Braw
    raw = torch.stack([t[:, :9].mean(1), t[:, 9:].mean(1)], 1)
    Bs = torch.stack([Bt[:, :9].sum(1), Bt[:, 9:].sum(1)], 1)
    part = torch.stack([t[:, :9].cumsum(1).abs().sum(1), t[:, 9:].cumsum(1).abs().sum(1)], 1)
    Braw = (Bs + U * (part + Bs)) / 9.0
    Braw = Braw + U * (raw.abs() + Braw)
    return z, Bz, raw, Braw


def hardnet_head(feat, w, bn_s, bn_sh):
    """tc_head_kernel on the layer-6 features feat [n,128,8,8] (one plane) with the head weights w [128,128,8,8] as stored: the descriptor
    [n,128] and its bound.  One accumulator over all 512 K = 16 steps (pixel by pixel, 16 channels a step); fmaf(d, scale, shift);
    the L2 norm from 128 fp32 fmafs, sqrtf, a division and a product (fewer than 140 roundings relative)."""
    n = feat.shape[0]
    fk = feat.reshape(n, 128, 64).transpose(1, 2).reshape(n, 64 * 8, 16)    # [n, step, 16]
    wk = w.reshape(128, 128, 64).transpose(1, 2).reshape(128, 64 * 8, 16)
    B = torch.zeros(n, 128, dtype=torch.float64, device=feat.device)
    S = torch.zeros_like(B)
    for t in range(0, 512, 64):   # chunks of steps keep the [n,128,steps] products small
        prod = torch.einsum("nsk,osk->nos", fk[:, t: t + 64], wk[:, t: t + 64])
        pa = torch.einsum("nsk,osk->nos", fk[:, t: t + 64].abs(), wk[:, t: t + 64].abs())
        Sc = S.unsqueeze(-1) + prod.cumsum(-1)
        B = B + C_ACC * 2.0 ** -23 * ((Sc - prod).abs() + pa).sum(-1) * MARGIN
        S = Sc[..., -1]
    v = S * bn_s + bn_sh
    Bv = B * bn_s.abs()
    Bv = Bv + U * (v.abs() + Bv)
    N = torch.sqrt((v * v).sum(1, keepdim=True) + 1e-8)
    d = v / N
    Bd = (Bv + d.abs() * Bv.norm(dim=1, keepdim=True)) / N + 140 * U * d.abs()
    return d, Bd


# ---- AffNet / OriNet outputs from the raw head outputs, bit for bit -------------------------------------------------------------
def rectify_up_is_up(a00, a01, a10, a11):
    """common.cuh rectify_up_is_up: one fp32 operation per torch operation, left to right, A[0,1] = 0 * det.  -> [n,4] fp32."""
    a00, a01, a10, a11 = (np.asarray(v, F32) for v in (a00, a01, a10, a11))
    with np.errstate(all="ignore"):
        det = np.sqrt(np.abs((a00 * a11 - a10 * a01) + F32(1e-10)))
        b2a2 = np.sqrt(a01 * a01 + a00 * a00)
        return np.stack([b2a2 / det, F32(0) * det, (a11 * a01 + a10 * a00) / (b2a2 * det), det / b2a2], 1).astype(F32)


# ---- float64 nets -----------------------------------------------------------------------------------------------------------------
def sd64(sd, device=None):
    return {k: (v.detach() if torch.is_tensor(v) else torch.from_numpy(np.asarray(v))).double().to(device) for k, v in sd.items()}


def input_norm64(P):
    flat = P.reshape(P.shape[0], -1)
    return (P - flat.mean(1).view(-1, 1, 1, 1)) / (flat.std(1).view(-1, 1, 1, 1) + 1e-7)


def trunk64(P, sd, kind):
    x = input_norm64(P)
    for i, (ci, co, s) in zip(CONV_IDX, cfg_of(kind)):
        x = F.conv2d(x, sd["features.%d.weight" % i], stride=s, padding=1)
        x = F.relu((x - sd["features.%d.running_mean" % (i + 1)].view(1, -1, 1, 1)) / torch.sqrt(sd["features.%d.running_var" % (i + 1)].view(1, -1, 1, 1) + 1e-5))
    return x


def net64(P, sd, kind):
    """The reference's forward in float64: AffNet A [n,2,2], OriNet angle [n], HardNet descriptors [n,128]."""
    x = trunk64(P, sd, kind)
    if kind == "affnet":
        t = torch.tanh(F.conv2d(x, sd["features.19.weight"], sd["features.19.bias"])).view(-1, 3)
        a00, a10, a11 = 1 + t[:, 0], t[:, 1], 1 + t[:, 2]
        det = torch.sqrt(torch.abs(a00 * a11 - a10 * 0 + 1e-10))
        b2a2 = torch.sqrt(a00 * a00)
        return torch.stack([b2a2 / det, 0 * det, (a10 * a00) / (b2a2 * det), det / b2a2], 1).view(-1, 2, 2)
    if kind == "orinet":
        m = torch.tanh(F.conv2d(x, sd["features.19.weight"], sd["features.19.bias"], padding=1)).mean(dim=(2, 3))
        return torch.atan2(m[:, 0] + 1e-8, m[:, 1] + 1e-8)
    x = F.conv2d(x, sd["features.19.weight"]).view(-1, 128)
    x = (x - sd["features.20.running_mean"]) / torch.sqrt(sd["features.20.running_var"] + 1e-5)
    return x / torch.sqrt((x * x).sum(1, keepdim=True) + 1e-8)


# ---- synthetic checkpoints -----------------------------------------------------------------------------------------------------------
def calibration_patches(seed=5, n=96):
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(n, 1, 8, 8, generator=g) * 255
    smooth = F.interpolate(base, size=(32, 32), mode="bilinear", align_corners=False)
    return (smooth + torch.rand(n, 1, 32, 32, generator=g) * 40).double()


def synthetic_state_dict(kind, seed, head_mult=1.0):
    """A seeded checkpoint with the reference's layout: He-normal conv weights times per-output-channel factors 2^U(-12, 2) and one all-zero
    channel per layer; BatchNorm running statistics calibrated in float64 on calibration patches (each layer's outputs have zero mean and
    their own variance, as a trained net's would); AffNet / OriNet head weights scaled so the pre-tanh values have a spread of 0.25 (|tanh| mostly below 0.76, as a trained AffNet's
    shapes stay near the identity); the HardNet
    head times head_mult, its BatchNorm calibrated after it."""
    g = torch.Generator().manual_seed(seed)
    x = input_norm64(calibration_patches())
    sd = {}
    for l, (i, (ci, co, s)) in enumerate(zip(CONV_IDX, cfg_of(kind))):
        w = torch.randn(co, ci, 3, 3, generator=g, dtype=torch.float64) * math.sqrt(2.0 / (9 * ci))
        w = w * torch.pow(2.0, torch.rand(co, generator=g, dtype=torch.float64) * 14 - 12).view(-1, 1, 1, 1)
        w[(7 * l + 3) % co] = 0
        w = w.float().double()
        z = F.conv2d(x, w, stride=s, padding=1)
        mean, var = z.mean(dim=(0, 2, 3)), z.var(dim=(0, 2, 3))
        sd["features.%d.weight" % i] = w.float()
        sd["features.%d.running_mean" % (i + 1)] = mean.float()
        sd["features.%d.running_var" % (i + 1)] = var.float()
        x = F.relu((z - mean.float().double().view(1, -1, 1, 1)) / torch.sqrt(var.float().double().view(1, -1, 1, 1) + 1e-5))
    c = cfg_of(kind)[-1][1]
    if kind == "hardnet":
        w = torch.randn(128, c, 8, 8, generator=g, dtype=torch.float64) * math.sqrt(1.0 / (64 * c)) * head_mult
        z = F.conv2d(x, w.float().double()).view(-1, 128)
        sd["features.19.weight"] = w.float()
        sd["features.20.running_mean"] = z.mean(0).float()
        sd["features.20.running_var"] = z.var(0).float()
    else:
        no = 3 if kind == "affnet" else 2
        w = torch.randn(no, c, 8, 8, generator=g, dtype=torch.float64)
        z = F.conv2d(x, w, padding=1 if kind == "orinet" else 0)
        w = w * (0.25 / z.std(dim=(0, 2, 3))).view(-1, 1, 1, 1)
        sd["features.19.weight"] = w.float()
        sd["features.19.bias"] = (torch.randn(no, generator=g, dtype=torch.float64) * 0.1).float()
    return sd


# ---- test patches ---------------------------------------------------------------------------------------------------------------------
IMPULSE_Y = (0, 1, 15, 16, 30, 31)
IMPULSE_X = (0, 1, 14, 15, 16, 17, 30, 31)


def edge_patches(seed=3):
    """Single-pixel impulses on a faint noise background at every (y, x) of the row ends, parities and the first kernel's warp split;
    x-checkerboards of period 1 and 2; constant 0 and 77; one low-contrast patch."""
    g = torch.Generator().manual_seed(seed)
    P = []
    for y in IMPULSE_Y:
        for x in IMPULSE_X:
            q = torch.rand(1, 1, 32, 32, generator=g) * 2
            q[0, 0, y, x] += 200.0
            P.append(q)
    xs = torch.arange(32)
    for period in (1, 2):
        P.append((((xs // period) % 2) * 255.0).float().view(1, 1, 1, 32).expand(1, 1, 32, 32).clone())
    P += [torch.zeros(1, 1, 32, 32), torch.full((1, 1, 32, 32), 77.0)]
    P.append(100.0 + torch.rand(1, 1, 32, 32, generator=g) * 0.05)
    return torch.cat(P)
