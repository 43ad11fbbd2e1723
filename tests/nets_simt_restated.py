"""The exact-fp32 SIMT net engine (ENGINE_SIMT, nets_simt.cu) restated one fp32 operation at a time, and a float64 forward with a
per-element error bound on every stage (test infrastructure, not product).

Every value the engine computes comes from a fixed sequence of fp32 operations, so its outputs are a function of the patches and the
weights alone.  `forward32` computes that function from float64 tensor operations on fp32 values, each rounded once to fp32 (for fp32
operands +, -, *, / and sqrt round correctly this way), with `fmaf32` for the fused steps.  It runs on the CPU or, in float64, on the
device.  The sequence, read off nets_simt.cu:
- weights: `nets_restated.fold` (BatchNorm folded in fp32 as ag_net_create does; HardNet's head shift is -mean / sqrt(var + eps));
- input normalisation (`conv3x3_kernel<.., NORM>`): thread t sums pixels t, t + 256, t + 512, t + 768 from 0; each warp reduces with an
  xor butterfly; the 8 warp sums are added in warp order from 0; mean = s / 1024; the same order for q = fmaf(d, d, q), d = v - mean;
  inv = 1 / (sqrtf(q / 1023) + 1e-7f); each staged pixel is (v - mean) * inv, the zero padding stays 0;
- `conv3x3_kernel`: acc = bias, then fmaf(x, w, acc) channel-major, tap-minor (tap = ky * 3 + kx), the padding included; fmaxf(acc, 0)
  (a NaN accumulator gives 0);
- AffNet head: lane l runs fmaf over k = l, l + 32, ... of 4096, a butterfly, 1 + tanhf(s + b), `rectify_up_is_up`;
- OriNet head: the same lane split against the 18 shifted copies of the 8x8 kernel (w_eff), a butterfly per output, m += tanhf(s + b)
  over the nine positions in order, m / 9, atan2f(m0 + 1e-8f, m1 + 1e-8f), cosf, sinf;
- HardNet head: one sequential fmaf chain per channel over k = 0..8191, v = fmaf(acc, scale, shift), a butterfly of v * v per warp,
  (w0 + w1) + (w2 + w3), v / sqrtf(ss + 1e-8f).
tanhf, atan2f, cosf and sinf are parameters (`Libm`): correctly rounded on the CPU, the device's own (ag_debug_tanhf, ag_debug_libm) in
the GPU tests.  `mut` names deliberate defects for the sensitivity tests (MUTATIONS).

The float64 side (`norm_bound`, `conv_bound`, the head bounds) gives each stage's value from the stage before it as the engine computed
it, and a bound on the engine's error: gamma_(k+1) (|b| + sum |w x|) for a chain of k FMAs (gamma_k = k u / (1 - k u), u = 2^-24), plus
2^-150 per FMA for results in the subnormal range; the normalisation and the heads are bounded the same way, operation by operation."""
import math

import numpy as np
import torch
import torch.nn.functional as F

import nets_restated as R
from scale_space_restated import fmaf32

U = 2.0 ** -24
ETA = 2.0 ** -150                       # largest error of one fp32 rounding in the subnormal range
FLT_MAX = float(np.finfo(np.float32).max)
EPS7, EPS8, EPS10 = (float(np.float32(v)) for v in (1e-7, 1e-8, 1e-10))
TANH_ULP, ATAN2_ULP, SINCOS_ULP = 2, 3, 2   # CUDA C++ Programming Guide, single-precision functions (full range)
MUTATIONS = ("tap_major", "contiguous_head", "pairwise_reduce", "norm_distributed", "unfused_affnet_head", "hardnet_shift_invstd",
             "pad_shift_row_end")


def gamma(k):
    return k * U / (1 - k * U)


def r32(x):
    """One fp32 rounding of float64 values."""
    return x.to(torch.float32).to(torch.float64)


def fma(a, b, c):
    return fmaf32(a, b, c).to(torch.float64)


class Libm:
    """The fp32 libm calls of the heads on float64 tensors of fp32 values.  Default: correctly rounded (float64 result rounded once)."""

    def tanhf(self, x):
        return r32(torch.tanh(x))

    def atan2f(self, y, x):
        return r32(torch.atan2(y, x))

    def cosf(self, x):
        return r32(torch.cos(x))

    def sinf(self, x):
        return r32(torch.sin(x))


def warp_sum(a, mut=()):
    """The warp's xor butterfly over the last axis (32 lanes), lane 0's sum; `pairwise_reduce`: adjacent pairs instead."""
    if "pairwise_reduce" in mut:
        while a.shape[-1] > 1:
            a = r32(a[..., 0::2] + a[..., 1::2])
        return a[..., 0]
    return R._butterfly(a, add=lambda x, y: r32(x + y))


def seq_sum(a):
    """s = 0; s += a[i] in order over the last axis."""
    s = torch.zeros_like(a[..., 0])
    for i in range(a.shape[-1]):
        s = r32(s + a[..., i])
    return s


# ---- weights ----------------------------------------------------------------------------------------------------------------------
def weights(sd, kind, device=None, mut=()):
    """fold() as float64 tensors: [(w [co,ci,3,3], b [co])] * 6 and the head (AffNet / OriNet: w, bias; HardNet: w, scale, shift)."""
    layers, head = R.fold(sd, kind)
    t = lambda a: torch.from_numpy(np.asarray(a, np.float32)).double().to(device)   # noqa: E731
    layers = [(t(w), t(b)) for w, b in layers]
    head = tuple(t(h) for h in head)
    if kind == "hardnet" and "hardnet_shift_invstd" in mut:
        g = lambda k: np.asarray(sd[k].detach().cpu().numpy() if torch.is_tensor(sd[k]) else sd[k], np.float32)   # noqa: E731
        m, v = g("features.20.running_mean"), g("features.20.running_var")
        head = (head[0], head[1], t((-m) * (np.float32(1) / np.sqrt(v + np.float32(1e-5)))))
    return layers, head


def orinet_weff(w):
    """ag_net_create's w_eff [4096, 18]: w_eff[ci*64 + y*8 + x][ch*9 + oy*3 + ox] = w[ch][ci][y - oy + 1][x - ox + 1], zero outside."""
    wp = F.pad(w, (1, 1, 1, 1))                                            # [2,64,10,10]
    return torch.stack([wp[ch, :, 2 - oy: 10 - oy, 2 - ox: 10 - ox] for ch in range(2) for oy in range(3) for ox in range(3)]).reshape(18, 4096).t()


# ---- the engine, one fp32 operation at a time -----------------------------------------------------------------------------------------
def input_norm(P, mut=()):
    """P [n,32,32] (float64 of fp32 values) -> the staged layer-1 input [n,32,32] and the per-patch (mean, q, inv)."""
    n = P.shape[0]
    v = P.reshape(n, 4, 256)                                               # pixel t + 256 j is v[:, j, t]
    s = seq_sum(v.transpose(1, 2))                                         # [n,256], thread t
    mean = r32(seq_sum(warp_sum(s.view(n, 8, 32), mut)) / 1024.0)
    q = torch.zeros_like(s)
    for j in range(4):
        d = r32(v[:, j] - mean[:, None])
        q = fma(d, d, q)
    q = seq_sum(warp_sum(q.view(n, 8, 32), mut))
    inv = r32(1.0 / r32(r32(torch.sqrt(r32(q / 1023.0))) + EPS7))
    m, i = mean.view(n, 1, 1), inv.view(n, 1, 1)
    if "norm_distributed" in mut:
        xn = r32(r32(P * i) - r32(m * i))
    else:
        xn = r32(r32(P - m) * i)
    return xn, (mean, q, inv)


def conv32(x, w, b, stride, mut=(), shift_row_end=False):
    """conv3x3_kernel: x [n,ci,H,H] -> fmaxf(acc, 0) [n,co,Ho,Ho]."""
    n, ci, H, _ = x.shape
    co, Ho = w.shape[0], H // stride
    xp = F.pad(x, (1, 1, 1, 1))
    acc = b.view(1, -1, 1, 1).expand(n, co, Ho, Ho).clone()
    order = [(c, t) for t in range(9) for c in range(ci)] if "tap_major" in mut else [(c, t) for c in range(ci) for t in range(9)]
    for c, t in order:
        ky, kx = divmod(t, 3)
        a = xp[:, c:c + 1, ky: ky + stride * Ho: stride, kx: kx + stride * Ho: stride]
        if shift_row_end and kx == 2:                                      # the row's first pixel in place of the right padding
            a = a.clone()
            a[..., -1] = xp[:, c:c + 1, ky: ky + stride * Ho: stride, 1]
        acc = fma(a, w[:, c, ky, kx].view(1, -1, 1, 1), acc)
    return torch.where(acc > 0, acc, torch.zeros_like(acc))               # fmaxf(acc, 0.f): NaN and -0 give +0


def lane_split(f, mut=()):
    """[n,4096] -> [n,128 steps,32 lanes]: lane l takes k = l + 32 j (`contiguous_head`: k = 128 l + j)."""
    n = f.shape[0]
    return f.view(n, 32, 128).transpose(1, 2) if "contiguous_head" in mut else f.view(n, 128, 32)


def affnet_head32(feat, w, bias, libm, mut=()):
    n = feat.shape[0]
    f = lane_split(feat.reshape(n, 4096), mut)                             # [n,128,32]
    wk = lane_split(w.reshape(3, 4096), mut)                               # [3,128,32]
    acc = torch.zeros(n, 3, 32, dtype=torch.float64, device=feat.device)
    for j in range(128):
        if "unfused_affnet_head" in mut:
            acc = r32(r32(f[:, None, j] * wk[None, :, j]) + acc)
        else:
            acc = fma(f[:, None, j], wk[None, :, j], acc)
    t = libm.tanhf(r32(warp_sum(acc, mut) + bias))                         # [n,3]
    a00, a10, a11 = r32(1.0 + t[:, 0]), t[:, 1], r32(1.0 + t[:, 2])
    raw = torch.stack([a00, a10, a11], 1)
    A = R.rectify_up_is_up(*(v.cpu().numpy() for v in (a00, torch.zeros_like(a00), a10, a11)))
    return raw, torch.from_numpy(A).double().to(feat.device)


def orinet_head32(feat, w, bias, libm, mut=()):
    n = feat.shape[0]
    f = lane_split(feat.reshape(n, 4096), mut)
    wk = lane_split(orinet_weff(w).t().contiguous(), mut)                  # [18,128,32]
    acc = torch.zeros(n, 18, 32, dtype=torch.float64, device=feat.device)
    for j in range(128):
        acc = fma(f[:, None, j], wk[None, :, j], acc)
    s = warp_sum(acc, mut)                                                 # [n,18]
    m0, m1 = torch.zeros_like(s[:, 0]), torch.zeros_like(s[:, 0])
    for o in range(9):
        m0 = r32(m0 + libm.tanhf(r32(s[:, o] + bias[0])))
        m1 = r32(m1 + libm.tanhf(r32(s[:, 9 + o] + bias[1])))
    m0, m1 = r32(m0 / 9.0), r32(m1 / 9.0)
    ang = libm.atan2f(r32(m0 + EPS8), r32(m1 + EPS8))
    c, sn = libm.cosf(ang), libm.sinf(ang)
    return torch.stack([m0, m1], 1), ang, torch.stack([c, sn, -sn, c], 1)


def hardnet_head32(feat, w, scale, shift, mut=()):
    n = feat.shape[0]
    f = feat.reshape(n, 8192)
    wk = w.reshape(128, 8192)
    acc = torch.zeros(n, 128, dtype=torch.float64, device=feat.device)
    for k in range(8192):
        acc = fma(f[:, k:k + 1], wk[None, :, k], acc)
    v = fma(acc, scale, shift)
    ss = warp_sum(r32(v * v).view(n, 4, 32), mut)                          # [n,4]
    ss = r32(r32(ss[:, 0] + ss[:, 1]) + r32(ss[:, 2] + ss[:, 3]))
    return r32(v / r32(torch.sqrt(r32(ss + EPS8)))[:, None])


def forward32(P, sd, kind, libm=None, mut=(), device=None):
    """The engine on patches P [n,1,32,32] (any float type; read as fp32).  -> dict: xn (staged layer-1 input), stats (mean, q, inv),
    layers [6 x [n,C,H,H]], and the outputs: AffNet raw (a00, a10, a11) and A [n,4]; OriNet raw (m0, m1), angle [n] and R [n,4];
    HardNet desc [n,128]."""
    libm = libm or Libm()
    P = torch.as_tensor(P).to(device=device, dtype=torch.float32).double().reshape(-1, 32, 32)
    layers, head = weights(sd, kind, P.device, mut)
    xn, stats = input_norm(P, mut)
    x, outs = xn.unsqueeze(1), []
    for l, ((w, b), (ci, co, s)) in enumerate(zip(layers, R.cfg_of(kind)), 1):
        x = conv32(x, w, b, s, mut, shift_row_end="pad_shift_row_end" in mut and l == 2)
        outs.append(x)
    r = {"xn": xn, "stats": stats, "layers": outs}
    if kind == "affnet":
        r["raw"], r["A"] = affnet_head32(x, *head, libm, mut)
    elif kind == "orinet":
        r["raw"], r["angle"], r["R"] = orinet_head32(x, *head, libm, mut)
    else:
        r["desc"] = hardnet_head32(x, *head, mut)
    return r


# ---- float64 values and bounds ---------------------------------------------------------------------------------------------------------
def norm_bound(P):
    """The float64 input normalisation (x - mean) / (std + 1e-7) of P [n,32,32] and a bound on the engine's staged value.  The bound is
    inf on patches where an fp32 intermediate can overflow (q = inf gives inv = 0) or that hold a NaN / inf."""
    P = P.double().reshape(-1, 32, 32)
    n = P.shape[0]
    flat = P.reshape(n, -1)
    M = flat.mean(1)
    Sd = flat.std(1)
    X = (P - M.view(n, 1, 1)) / (Sd.view(n, 1, 1) + 1e-7)
    D = (flat - M[:, None]).abs()
    Q = (D * D).sum(1)
    # depth of the adds: 3 in the thread, 5 in the butterfly, 7 over the warps, and one fmaf per term of q
    e_m = gamma(16) * flat.abs().sum(1) / 1024 + ETA
    e_d = e_m[:, None] + U * (D + e_m[:, None])                            # per pixel
    e_dd = (2 * D * e_d + e_d * e_d).sum(1)
    e_q = gamma(16) * (Q + e_dd) + e_dd + 1024 * ETA
    e_1 = e_q / 1023 + U * (Q + e_q) / 1023 + ETA
    e_sd = torch.minimum(torch.sqrt(e_1), e_1 / Sd) + U * (Sd + torch.sqrt(e_1))
    e_c = abs(EPS7 - 1e-7)
    Den = Sd + 1e-7
    e_den = e_sd + e_c + U * (Den + e_sd + e_c)
    e_inv = torch.where(e_den < Den, e_den / (Den * (Den - e_den).clamp(min=1e-300)), torch.full_like(Den, math.inf))
    e_inv = e_inv + U * (1 / Den + e_inv)
    B = e_d.view(n, 32, 32) * (1 / Den + e_inv).view(n, 1, 1) + D.view(n, 32, 32) * e_inv.view(n, 1, 1)
    B = B + U * (X.abs() + B) + ETA
    bad = ~torch.isfinite(flat).all(1) | ((Q + e_q) * (1 + gamma(20)) >= FLT_MAX) | (flat.abs().sum(1) * (1 + gamma(20)) >= FLT_MAX)
    B[bad] = math.inf
    return X, B


def conv_bound(x, w, b, stride):
    """The pre-ReLU float64 value of conv3x3_kernel on the engine's input x and a bound on the engine's accumulator: a chain of
    k = 9 ci FMAs from the bias, gamma_(k+1) (|b| + sum |w x|) + k 2^-150."""
    k = 9 * x.shape[1]
    y = F.conv2d(x, w, b, stride=stride, padding=1)
    Pabs = F.conv2d(x.abs(), w.abs(), b.abs(), stride=stride, padding=1)
    return y, gamma(k + 1) * Pabs * R.MARGIN + k * ETA


def _spacing(t):
    return torch.clamp(R.ulp(t, "fp32"), min=2.0 ** -149)


def _widen(lo, hi):
    return lo - U * lo.abs() - ETA, hi + U * hi.abs() + ETA


def _imul(a, b):
    p = torch.stack([a[0] * b[0], a[0] * b[1], a[1] * b[0], a[1] * b[1]])
    return _widen(p.min(0).values, p.max(0).values)


def _idiv(a, b):
    ok = (b[0] > 0) | (b[1] < 0)
    inv = (1 / torch.where(ok, b[1], torch.ones_like(b[1])), 1 / torch.where(ok, b[0], torch.ones_like(b[0])))
    p = torch.stack([a[0] * inv[0], a[0] * inv[1], a[1] * inv[0], a[1] * inv[1]])
    lo, hi = _widen(p.min(0).values, p.max(0).values)
    return torch.where(ok, lo, torch.full_like(lo, -math.inf)), torch.where(ok, hi, torch.full_like(hi, math.inf))


def _iabs(a):
    lo = torch.where((a[0] <= 0) & (a[1] >= 0), torch.zeros_like(a[0]), torch.minimum(a[0].abs(), a[1].abs()))
    return lo, torch.maximum(a[0].abs(), a[1].abs())


def _isqrt(a):
    return _widen(torch.sqrt(a[0].clamp(min=0)), torch.sqrt(a[1].clamp(min=0)))


def affori_head_bound(feat, w, bias, kind):
    """The float64 head on the engine's layer-6 features: AffNet raw (1 + tanh, tanh, 1 + tanh) and OriNet (m0, m1) [n,2..3] with their
    bound.  Each dot product is 128 FMAs per lane and a 5-level butterfly, then the bias: gamma_134; tanhf within TANH_ULP ulp."""
    n = feat.shape[0]
    f = feat.reshape(n, 4096)
    wk = w.reshape(3, 4096) if kind == "affnet" else orinet_weff(w).t()
    bb = bias if kind == "affnet" else bias.repeat_interleave(9)
    z = f @ wk.t() + bb
    Bz = gamma(134) * (f.abs() @ wk.abs().t() + bb.abs()) * R.MARGIN + 128 * ETA
    t = torch.tanh(z)
    Bt = Bz + TANH_ULP * _spacing(t)
    if kind == "affnet":
        raw = torch.stack([1 + t[:, 0], t[:, 1], 1 + t[:, 2]], 1)
        return raw, Bt + U * (raw.abs() + Bt)
    m = torch.stack([t[:, :9].mean(1), t[:, 9:].mean(1)], 1)
    Bs = torch.stack([Bt[:, :9].sum(1), Bt[:, 9:].sum(1)], 1)
    ta = torch.stack([t[:, :9].abs().sum(1), t[:, 9:].abs().sum(1)], 1)
    Bm = (Bs + gamma(8) * (ta + Bs)) / 9
    return m, Bm + U * (m.abs() + Bm) + ETA


def affnet_A_interval(raw, Braw):
    """The interval each element of A [n,4] lies in when (a00, a10, a11) lie within raw +- Braw and every fp32 operation of
    rectify_up_is_up rounds outward (a01 = 0)."""
    a00, a10, a11 = ((raw[:, i] - Braw[:, i], raw[:, i] + Braw[:, i]) for i in range(3))
    p = _imul(a00, a11)
    e_c = abs(EPS10 - 1e-10)
    det = _isqrt(_iabs(_widen(p[0] + EPS10 - e_c, p[1] + EPS10 + e_c)))
    b2a2 = _isqrt(_widen(*_sq(a00)))
    A0 = _idiv(b2a2, det)
    A2 = _idiv(_imul(a10, a00), _imul(b2a2, det))
    A3 = _idiv(det, b2a2)
    z = torch.zeros_like(raw[:, 0])
    lo = torch.stack([A0[0], z, A2[0], A3[0]], 1)
    hi = torch.stack([A0[1], z, A2[1], A3[1]], 1)
    return lo, hi


def _sq(a):
    lo, hi = _iabs(a)
    return lo * lo, hi * hi


def orinet_angle_bound(m, Bm):
    """The float64 angle atan2(m0 + 1e-8, m1 + 1e-8) and a bound on the engine's: the box (m0, m1) +- Bm (plus the two fp32 adds) seen from
    the origin, and atan2f within ATAN2_ULP ulp.  pi where the box holds the origin."""
    y, x = m[:, 0] + 1e-8, m[:, 1] + 1e-8
    By = Bm[:, 0] + U * (y.abs() + Bm[:, 0]) + abs(EPS8 - 1e-8) + ETA
    Bx = Bm[:, 1] + U * (x.abs() + Bm[:, 1]) + abs(EPS8 - 1e-8) + ETA
    ang = torch.atan2(y, x)
    rho, r = torch.sqrt(By * By + Bx * Bx), torch.sqrt(y * y + x * x)
    d = torch.where(rho < r, torch.asin((rho / r).clamp(max=1.0)), torch.full_like(r, math.pi))
    return ang, d * R.MARGIN + ATAN2_ULP * 2.0 ** -22


def hardnet_head_bound(feat, w, scale, shift):
    """The float64 descriptor on the engine's layer-6 features and its bound: 8192-FMA chains (gamma_8192), fmaf(acc, scale, shift), and the
    L2 norm (v * v, 7 adds, + 1e-8f, sqrtf, a division: under 8 roundings relative)."""
    n = feat.shape[0]
    f = feat.reshape(n, 8192)
    wk = w.reshape(128, 8192)
    acc = f @ wk.t()
    Bacc = gamma(8192) * (f.abs() @ wk.abs().t()) * R.MARGIN + 8192 * ETA
    v = acc * scale + shift
    Bv = Bacc * scale.abs()
    Bv = Bv + U * (v.abs() + Bv) + ETA
    N = torch.sqrt((v * v).sum(1, keepdim=True) + 1e-8)
    d = v / N
    Bd = (Bv + d.abs() * Bv.norm(dim=1, keepdim=True)) / N * R.MARGIN + 8 * U * d.abs() + ETA
    return d, Bd


def wrap(d):
    """An angle difference in (-pi, pi]."""
    return torch.atan2(torch.sin(d), torch.cos(d))


# ---- checks ------------------------------------------------------------------------------------------------------------------------
def check_within(tag, err, B):
    """err <= B wherever the bound is finite; prints the worst ratio."""
    m = torch.isfinite(B) & torch.isfinite(err)
    ratio = (err[m] / B[m]).max().item() if m.any() else 0.0
    print("%s: max err/bound %.3f (max err %.2e, %d unbounded)" % (tag, ratio, err[m].max().item() if m.any() else 0.0, int((~m).sum())))
    bad = m & (err > B)
    assert not bad.any(), "%s: %d elements beyond the bound, first %s" % (tag, int(bad.sum()), bad.nonzero()[0].tolist())
    return ratio


def check_bounds(tag, kind, sd, P, layers, outs, restated=None):
    """Every stage of the engine within its float64 bound, from the engine's previous stage: the staged input (restated, `restated["xn"]`
    when given), layers 1-6, the head (AffNet: the raw head within its bound, A inside its interval; OriNet: (m0, m1) and the angle;
    HardNet: descriptors).  Returns the worst ratios."""
    dev = layers[0].device
    w, head = weights(sd, kind, dev)
    Pd = P.to(dev).double().reshape(-1, 32, 32)
    xn = restated["xn"] if restated is not None else input_norm(Pd)[0]
    X, BX = norm_bound(Pd)
    worst = {"norm": check_within("%s input norm" % tag, (xn - X).abs(), BX)}
    x = xn.unsqueeze(1)
    for l, ((wl, bl), (ci, co, s)) in enumerate(zip(w, R.cfg_of(kind)), 1):
        y, B = conv_bound(x, wl, bl, s)
        worst["layer %d" % l] = check_within("%s layer %d" % (tag, l), (layers[l - 1] - y.clamp(min=0)).abs(), B)
        x = layers[l - 1]
    if kind == "hardnet":
        d64, Bd = hardnet_head_bound(x, *head)
        worst["head"] = check_within("%s head" % tag, (outs["desc"] - d64).abs(), Bd)
        return worst
    raw64, Braw = affori_head_bound(x, *head, kind)
    if restated is not None:
        worst["raw head"] = check_within("%s raw head (restated, bit-exact)" % tag, (restated["raw"] - raw64).abs(), Braw)
    if kind == "affnet":
        lo, hi = affnet_A_interval(raw64, Braw)
        A = outs["A"]
        inside = (A >= lo) & (A <= hi)
        m = torch.isfinite(lo) & torch.isfinite(hi)
        print("%s A: inside its interval %d / %d (%d unbounded), widest %.2e" % (tag, int((inside & m).sum()), int(m.sum()), int((~m).sum()),
                                                                                (hi - lo)[m].max().item()))
        assert (inside | ~m).all(), tag
    else:
        a64, Ba = orinet_angle_bound(raw64, Braw)
        worst["angle"] = check_within("%s angle" % tag, wrap(outs["angle"] - a64).abs(), Ba)
    return worst


# ---- the normalisation's edges ---------------------------------------------------------------------------------------------------------
SPECIAL = ("zero", "constant", "times 2^60", "times 2^-70", "times 2^-120", "NaN pixel", "+inf pixel", "-inf pixel")


def special_patches(seed=17):
    """The input normalisation's edges, in SPECIAL's order: all zero and constant (q = 0, inv = 1 / 1e-7f); seeded 0..255 noise times 2^60
    (q overflows to inf, inv = 0), times 2^-70 (products d * d and partial sums of q in the subnormal range) and times 2^-120 (every d * d
    underflows, q = 0); one NaN, +inf and -inf pixel."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(1, 1, 32, 32, generator=g) * 255
    P = [torch.zeros(1, 1, 32, 32), torch.full((1, 1, 32, 32), 77.0), base * 2.0 ** 60, base * 2.0 ** -70, base * 2.0 ** -120]
    for y, x, v in ((3, 31, math.nan), (16, 0, math.inf), (31, 17, -math.inf)):
        q = torch.rand(1, 1, 32, 32, generator=g) * 255
        q[0, 0, y, x] = v
        P.append(q)
    return torch.cat(P).float()
