"""CPU tests of the float64 net restatement (tests/nets_restated.py): its rounding helpers against torch, its nets against the oracle and
the goldens, and its sensitivity.  An emulation of the engine (exact operands, accumulation perturbed within the model, stores rounded)
passes the per-element checks; each mutation of it that a kernel bug would cause fails them."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import affnet_oracle as O
import nets_restated as R
from helpers import gold, load_weights

W = load_weights()


# ---- rounding helpers ------------------------------------------------------------------------------------------------------------
def _specials(fmt):
    p, emin = R.FMT[fmt]
    g = torch.Generator().manual_seed(1)
    e = torch.randint(emin - p - 2, 16, (20000,), generator=g).double()
    v = (torch.rand(20000, generator=g, dtype=torch.float64) + 1) * torch.pow(2.0, e) * torch.where(torch.rand(20000, generator=g) < 0.5, -1.0, 1.0)
    ties = []                                  # exact midpoints between neighbours, normal and subnormal
    for ex in (emin - p + 1, emin - 3, emin, -1, 0, 3):
        k = torch.arange(1, 64, dtype=torch.float64)
        ties.append((k + 0.5) * 2.0 ** ex)
    return torch.cat([v.float().double(), torch.cat(ties).float().double()])


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_rounding_equals_torch(fmt):
    v = _specials(fmt)
    ref = (v.float().half() if fmt == "fp16" else v.float().bfloat16()).double()
    assert torch.equal(R.rnd(v, fmt), ref)
    hi, lo = R.split(v, fmt)
    hr = ref
    lr = ((v.float() - hr.float()).half() if fmt == "fp16" else (v.float() - hr.float()).bfloat16()).double()
    assert torch.equal(hi, hr) and torch.equal(lo, lr)


def test_input_norm32_matches_oracle():
    P = torch.cat([torch.from_numpy(gold("graf_crop.npz")["aff_patches"]), R.edge_patches()])
    x = R.input_norm32(P.numpy())
    ref = O.input_norm(P).numpy()[:, 0]
    scale = np.abs(ref).max(axis=(1, 2), keepdims=True) + 1e-30
    assert (np.abs(x - ref) / scale).max() < 4e-6
    for c in (0.0, 77.0):                       # exactly constant patches give exact zeros
        assert not np.any(R.input_norm32(np.full((1, 32, 32), c, np.float32)))


@pytest.mark.parametrize("kind", ["affnet", "orinet", "hardnet"])
def test_net64_matches_oracle_and_goldens(kind):
    """The float64 nets against the reference's outputs on the shipped weights (nets_random.npz, the TorchScript raw heads of jit.npz) and
    against the fp32 oracle on the graf crop's patches."""
    z = gold("nets_random.npz")
    P = torch.from_numpy(z["patches"])
    out = R.net64(P.double(), R.sd64(W[kind]), kind)
    golden = {"affnet": "affnet_A", "orinet": "orinet_angle", "hardnet": "hardnet_desc"}[kind]
    ref = torch.from_numpy(z[golden]).double()
    assert (out - ref).abs().max() < 2e-5, (out - ref).abs().max()
    # shipped weights against the fp32 oracle
    P = torch.from_numpy(gold("graf_crop.npz")["aff_patches"])
    fo = {"affnet": O.affnet_forward, "orinet": O.orinet_angle, "hardnet": O.hardnet_forward}[kind]
    assert (R.net64(P.double(), R.sd64(W[kind]), kind) - fo(P, W[kind]).double()).abs().max() < 2e-5
    if kind != "hardnet":
        zj = gold("jit.npz")
        Pj = torch.from_numpy(zj["patches"]).double()
        x = R.trunk64(Pj, R.sd64(W[kind]), kind)
        sdd = R.sd64(W[kind])
        t = torch.tanh(F.conv2d(x, sdd["features.19.weight"], sdd["features.19.bias"], padding=1 if kind == "orinet" else 0))
        raw = t.mean(dim=(2, 3)) if kind == "orinet" else t.view(-1, 3) + torch.tensor([1.0, 0.0, 1.0], dtype=torch.float64)
        assert (raw - torch.from_numpy(zj[kind + "_raw"]).double()).abs().max() < 2e-5


def test_rectify_matches_oracle():
    """rectify_up_is_up equals the reference's expression with every operation correctly rounded to fp32 (each float64 operation on fp32
    operands, rounded once), and the oracle's torch arithmetic within 4 ulp (torch's CPU fp32 sqrt is not always correctly rounded)."""
    g = torch.Generator().manual_seed(4)
    a = ((torch.rand(4000, 3, generator=g) * 2 - 1) * 0.9).numpy()
    f = lambda v: np.float64(np.float32(v)) if np.isscalar(v) else v.astype(np.float32).astype(np.float64)
    a00, a10, a11 = f(1 + a[:, 0].astype(np.float32)), f(a[:, 1]), f(1 + a[:, 2].astype(np.float32))
    det = f(np.sqrt(np.abs(f(f(a00 * a11) + np.float64(np.float32(1e-10))))))
    b2a2 = f(np.sqrt(f(0.0 + f(a00 * a00))))
    ref = np.stack([f(b2a2 / det), 0 * det, f(f(0.0 + f(a10 * a00)) / f(b2a2 * det)), f(det / b2a2)], 1).astype(np.float32)
    out = R.rectify_up_is_up(a00, np.zeros(4000, np.float32), a10, a11)
    assert np.array_equal(out.view(np.int32), ref.view(np.int32))
    A = torch.zeros(4000, 2, 2)
    A[:, 0, 0] = torch.from_numpy(a00).float(); A[:, 1, 0] = torch.from_numpy(a10).float(); A[:, 1, 1] = torch.from_numpy(a11).float()
    o = O.rectify_up_is_up(A).numpy().reshape(-1, 4)
    assert np.all(np.abs(o - out) <= 4 * np.spacing(np.abs(out)))


# ---- emulation of the engine and its mutations -------------------------------------------------------------------------------------
def _emulate(y, B, fmt, pair, seed, rz=False):
    """The engine's stored output: the exact value moved by up to half the bound, ReLU, then the store (hi + lo, or one plane)."""
    g = torch.Generator().manual_seed(seed)
    v = torch.clamp(y + 0.5 * B * (torch.rand(y.shape, generator=g, dtype=torch.float64) * 2 - 1), min=0)
    if pair:
        hi, lo = R.split(v.float().double(), "fp16")
        return hi + lo
    return (R.rnd_rz if rz else R.rnd)(v.float().double(), fmt)


def _passes(out, y, B, fmt, pair):
    if pair:
        return bool(((out - torch.clamp(y, min=0)).abs() <= R.pair_store_bound(y, B)).all())
    lo, hi = R.admissible(y, B, fmt)
    return bool(((out >= lo) & (out <= hi)).all())


def _patches():
    g = torch.Generator().manual_seed(8)
    return torch.cat([torch.from_numpy(gold("graf_crop.npz")["aff_patches"])[:6], R.edge_patches()[::5], torch.rand(3, 1, 32, 32, generator=g) * 255])


def _tap_only(w, dx):
    m = torch.zeros_like(w)
    m[..., dx] = w[..., dx]
    return m


MUTATIONS = ["none", "hardnet_no_residual_l2", "hardnet_no_residual_l3", "affnet_no_alo_whi", "right_dropped_x0", "left_dropped_x31",
             "pair_partner_neighbour", "neighbour_channel_bias", "round_toward_zero_store"]


@pytest.mark.parametrize("mutation", MUTATIONS)
@pytest.mark.parametrize("ckpt", ["shipped", "synthetic"])
def test_emulated_engine(mutation, ckpt):
    """Layers 1-6 of an emulated engine, each from the emulation's previous layer.  The unmutated emulation passes every layer; every
    mutation fails at least one."""
    kind = "hardnet" if mutation.startswith("hardnet") or mutation == "round_toward_zero_store" else "affnet"
    sd = W[kind] if ckpt == "shipped" else R.synthetic_state_dict(kind, 13 if kind == "hardnet" else 11)
    fmt, pair = "fp16", kind != "hardnet"
    ops, _ = R.operands(kind, sd)
    cfg = R.cfg_of(kind)
    P = _patches()
    y1, B1 = R.layer1(P, *ops[0], fmt)
    x_ref, xr = R.store_interval(y1, B1, fmt, pair)
    x = _emulate(y1, B1, fmt, pair, 0)
    ok = True
    for l in range(2, 7):
        w_hi, w_lo, b = ops[l - 1]
        s = cfg[l - 1][2]
        if l > 2:
            x_ref, xr = x, None
        y, B = R.conv_layer(x_ref, w_hi, w_lo, b, s, xr=xr, a_lo=R.a_lo_of(x_ref) if pair else None)
        ym = F.conv2d(x, w_hi + w_lo, stride=s, padding=1) + b.view(1, -1, 1, 1)      # the emulated engine's exact value
        if mutation == "hardnet_no_residual_l%d" % l:
            ym = ym - F.conv2d(x, w_lo, stride=s, padding=1)
        if mutation == "affnet_no_alo_whi" and l == 4:
            ym = ym - F.conv2d(x - R.rnd(x, "fp16"), w_hi, stride=s, padding=1)
        if mutation == "right_dropped_x0" and l == 2:
            ym[..., 0] -= F.conv2d(x, _tap_only(w_hi + w_lo, 2), padding=1)[..., 0]
        if mutation == "left_dropped_x31" and l == 2:
            ym[..., -1] -= F.conv2d(x, _tap_only(w_hi + w_lo, 0), padding=1)[..., -1]
        if mutation == "pair_partner_neighbour" and l == 6:   # x = 0's left neighbour from x = 7 of the other patch of the pair unit
            partner = x[torch.arange(x.shape[0]) ^ 1 if x.shape[0] % 2 == 0 else torch.arange(x.shape[0])]
            ym[..., 0] += F.conv2d(partner[..., 7:8], (w_hi + w_lo)[..., 0:1], padding=(1, 0))[..., 0]
        if mutation == "neighbour_channel_bias" and l == 5:
            ym = ym - b.view(1, -1, 1, 1) + b[torch.arange(b.numel()) ^ 1].view(1, -1, 1, 1)
        x = _emulate(ym, B, fmt, pair, l, rz=mutation == "round_toward_zero_store" and l == 3)
        ok = ok and _passes(x, y, B, fmt, pair)
    assert ok == (mutation == "none"), (mutation, ckpt)


def test_small_head_needs_the_power_of_two_scale():
    """HardNet head weights 2^-10 of the shipped scale (BatchNorm recalibrated): stored as plain fp16 they are subnormals and the descriptors
    miss the 6e-4 contract; with the power-of-two scale of every other layer they meet it."""
    sd = R.synthetic_state_dict("hardnet", 13, head_mult=2.0 ** -10)
    P = torch.cat([torch.from_numpy(gold("graf_crop.npz")["ori_desc_patches"])[:48], _patches()]).double()
    s64 = R.sd64(sd)
    ref = R.net64(P, s64, "hardnet")
    feat = R.rnd(R.trunk64(P, s64, "hardnet"), "fp16")
    _, head = R.operands("hardnet", sd)
    w = torch.from_numpy(R.fold(sd, "hardnet")[1][0]).double()

    def desc(wr):
        v = F.conv2d(feat, wr).view(-1, 128) * head[2] + head[3]
        return v / torch.sqrt((v * v).sum(1, keepdim=True) + 1e-8)
    plain = (desc(R.rnd(w, "fp16")) - ref).abs().max().item()
    scaled = (desc(head[0]) - ref).abs().max().item()
    print("\nsmall head: plain fp16 %.2e, scaled %.2e" % (plain, scaled))
    assert plain > 6e-4 and scaled < 3e-4
