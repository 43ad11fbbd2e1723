"""GPU tests of the exact-fp32 SIMT net engine (ENGINE_SIMT, nets_simt.cu) against its restatement (tests/nets_simt_restated.py).

Every output (AffNet A, OriNet angle and R, HardNet descriptors; through the Python modules and through the C ABI) and every conv layer
(ag_debug_tcx_layer under ENGINE_SIMT) must be bit-identical to the restatement run on the device in float64 with the device's own tanhf
(ag_debug_tanhf), atan2f, cosf and sinf (ag_debug_libm); NaN positions must match.  Every element must also lie within its float64 bound,
each stage computed from the engine's own previous stage; the worst error / bound per layer and head is printed.  Checkpoints: the
shipped weights, the seeded synthetic ones of nets_restated.synthetic_state_dict and the HardNet small-head one.  Patches: the 257 of
test_gpu_net_bounds.patches() and the normalisation's edges (nets_simt_restated.special_patches)."""
import subprocess

import numpy as np
import pytest
import torch

import nets_restated as R
import nets_simt_restated as S
from helpers import SENTINEL, net_forward_rows
from test_gpu_handcrafted import probe, same, ulps
from test_gpu_net_bounds import CKPTS, patches, state_dict
from test_gpu_tcx_rowends import rowend_patches

pytestmark = pytest.mark.gpu
DEV = "cuda"
BATCHES = (1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 257)


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("\n%s; nvidia-smi: %s" % (torch.cuda.get_device_name(), q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "n/a"))
    return lib


def tanhf_probe(L, x):
    """ag_debug_tanhf on an fp32 array -> numpy."""
    dx = torch.from_numpy(np.ascontiguousarray(x, np.float32).ravel()).to(DEV)
    dy = torch.full_like(dx, SENTINEL)
    L.check(L.lib().ag_debug_tanhf(L.ptr(dx), dx.numel(), L.ptr(dy), L.stream_ptr()))
    torch.cuda.synchronize()
    return dy.cpu().numpy().reshape(np.shape(x))


class DeviceLibm(S.Libm):
    """The device's tanhf, atan2f, cosf and sinf on float64 tensors of fp32 values."""

    def __init__(self, L):
        self.L = L

    def _f(self, fn, *xs):
        out = fn(*(x.float().cpu().numpy() for x in xs))
        return torch.from_numpy(np.asarray(out, np.float32)).double().to(xs[0].device)

    def tanhf(self, x):
        return self._f(lambda a: tanhf_probe(self.L, a), x)

    def atan2f(self, y, x):
        return self._f(lambda a, b: probe(self.L, a, b)[0], y, x)

    def cosf(self, x):
        return self._f(lambda a: probe(self.L, np.zeros_like(a), a)[1], x)

    def sinf(self, x):
        return self._f(lambda a: probe(self.L, np.zeros_like(a), a)[2], x)


def module(L, kind, sd):
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    m = {"affnet": lambda: AffNetFast(PS=32), "orinet": lambda: OriNetFast(PS=32), "hardnet": HardNet}[kind]()
    m.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    m = m.eval().to(DEV)
    m.set_engine(L.ENGINE_SIMT)
    return m


def all_patches():
    return torch.cat([patches(), S.special_patches()]).contiguous()


def layer_out(L, net, P, upto):
    """Conv layer `upto` (1..6) of the SIMT trunk, fp32 NCHW, through ag_debug_tcx_layer."""
    lib = L.lib()
    n = P.size(0)
    ci, co, s = R.cfg_of({L.NET_AFFNET: "affnet", L.NET_ORINET: "orinet", L.NET_HARDNET: "hardnet"}[net.KIND])[upto - 1]
    H = 32 // (2 if upto >= 3 else 1) // (2 if upto >= 5 else 1)
    ws_bytes = lib.ag_net_workspace_bytes(net.KIND, n)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    out = torch.full((n, co, H, H), SENTINEL, device=DEV)
    Pd = P.to(DEV).contiguous()
    L.check(lib.ag_debug_tcx_layer(net.handle(), L.ptr(Pd), n, upto, L.ptr(out), L.ptr(ws), ws_bytes, L.stream_ptr()))
    torch.cuda.synchronize()
    return out.double()


def outputs(L, net, kind, P):
    """The engine's outputs through the modules and through the C ABI, as float64 on the device."""
    Pd = P.to(DEV)
    if kind == "affnet":
        out, _ = net_forward_rows(L, net, P)
        return {"A": net(Pd).reshape(-1, 4).double(), "A (C ABI)": out.reshape(-1, 4).double()}
    if kind == "orinet":
        out, ang = net_forward_rows(L, net, P)
        return {"angle": net(Pd, return_rot_matrix=False).double(), "R": net(Pd).reshape(-1, 4).double(),
                "angle (C ABI)": ang.double(), "R (C ABI)": out.reshape(-1, 4).double()}
    out, _ = net_forward_rows(L, net, P)
    return {"desc": net(Pd).double(), "desc (C ABI)": out.double()}


def bits(a, b):
    return same(a.float().cpu().numpy(), b.float().cpu().numpy())


def first_diff(a, b):
    a, b = a.float().cpu().numpy(), b.float().cpu().numpy()
    d = np.argwhere(~((a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))))
    i = tuple(d[0])
    return "%d differ, first %s: engine %r restated %r" % (len(d), i, a[i], b[i])


# ---- the tanhf probe --------------------------------------------------------------------------------------------------------------------
def test_tanhf_probe_within_documented_ulps(L):
    rng = np.random.default_rng(7)
    n = 1 << 20
    mag = np.float32(10.0) ** rng.uniform(-46, 38.5, n).astype(np.float32)      # every binade, subnormals included
    sgn = np.where(rng.random(n) < 0.5, -1.0, 1.0).astype(np.float32)
    x = np.concatenate([sgn * mag, rng.uniform(-12, 12, n).astype(np.float32)]).astype(np.float32)
    with np.errstate(all="ignore"):
        e = ulps(tanhf_probe(L, x), np.tanh(x.astype(np.float64)))
    print("\ntanhf probe: %.2f ulp max over %d points" % (e.max(), x.size))
    assert e.max() <= S.TANH_ULP, (e.max(), x[np.argmax(e)])


def test_tanhf_probe_special_values(L):
    tiny = np.float32(1e-45)
    x = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, tiny, -tiny, np.float32(1.1e-38), np.float32(-5e-39)], np.float32)
    y = tanhf_probe(L, x)
    assert same(y[:4], np.array([0.0, -0.0, 1.0, -1.0], np.float32)) and np.isnan(y[4])
    assert (ulps(y[5:], np.tanh(x[5:].astype(np.float64))) <= S.TANH_ULP).all()
    sat = np.concatenate([np.linspace(8.0, 10.0, 4097, dtype=np.float32), np.float32(9.01) + np.arange(-64, 65, dtype=np.float32) * np.spacing(np.float32(9))])
    sat = np.concatenate([sat, -sat]).astype(np.float32)
    ys = tanhf_probe(L, sat)
    es = ulps(ys, np.tanh(sat.astype(np.float64)))
    print("\ntanhf near saturation: %.2f ulp max, tanhf == +-1 from |x| = %g" % (es.max(), np.abs(sat[np.abs(ys) == 1]).min()))
    assert es.max() <= S.TANH_ULP and (np.abs(ys) <= 1).all()


# ---- bit for bit and within the bounds --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ckpt", CKPTS)
@pytest.mark.parametrize("kind", ["affnet", "orinet", "hardnet"])
def test_simt_bit_exact_and_bounded(L, kind, ckpt):
    if ckpt == "hardnet_small_head" and kind != "hardnet":
        pytest.skip("the small-head checkpoint is a HardNet variant")
    sd = state_dict(kind, ckpt)
    net = module(L, kind, sd)
    P = all_patches()
    tag = "%s %s" % (kind, ckpt)
    r = S.forward32(P, sd, kind, DeviceLibm(L), device=DEV)
    layers = [layer_out(L, net, P, l) for l in range(1, 7)]
    for l in range(6):
        assert bits(layers[l], r["layers"][l]), "%s layer %d: %s" % (tag, l + 1, first_diff(layers[l], r["layers"][l]))
    outs = outputs(L, net, kind, P)
    for name, v in outs.items():
        ref = r[name.split(" ")[0]]
        assert bits(v, ref), "%s %s: %s" % (tag, name, first_diff(v, ref))
    print()
    S.check_bounds(tag, kind, sd, P, layers, outs, r)
    # end to end against the float64 reference on the natural patches (the graf crops and the seeded noise)
    n_noise = 257 - 96 - rowend_patches().size(0) - R.edge_patches().size(0)
    sel = torch.cat([torch.arange(96), torch.arange(257 - n_noise, 257)])
    ref = R.net64(P[sel].double().to(DEV), R.sd64(sd, DEV), kind)
    sel = sel.to(DEV)
    if kind == "orinet":
        e = S.wrap(outs["angle"][sel] - ref).abs()
    else:
        e = (outs["A" if kind == "affnet" else "desc"][sel] - ref.reshape(len(sel), -1)).abs()
    print("%s end to end vs float64 (natural patches): max err %.2e" % (tag, e.max().item()))
    assert e.max().item() < {"affnet": 5e-5, "orinet": 1e-4, "hardnet": 6e-4}[kind]


@pytest.mark.parametrize("kind", ["affnet", "orinet", "hardnet"])
def test_simt_batch_sizes(L, kind):
    """n = 1..5 (OriNet's 4 patches per warp and its min(p0 + q, n - 1) clamp), 7..9 (AffNet's 8 per CTA), 15..17 (HardNet's 16 per CTA,
    zero-filled rows), 31..33 (OriNet's 32 per CTA) and 257: every patch gets the bits of the full batch, which
    test_simt_bit_exact_and_bounded pins to the restatement; layer 6 too."""
    net = module(L, kind, state_dict(kind, "shipped"))
    P = all_patches()
    full, full6 = outputs(L, net, kind, P), layer_out(L, net, P, 6)
    for n in BATCHES:
        part = outputs(L, net, kind, P[:n].contiguous())
        for name, v in part.items():
            assert bits(v, full[name][:n]), (kind, n, name)
        assert bits(layer_out(L, net, P[:n].contiguous(), 6), full6[:n]), (kind, n)


@pytest.mark.parametrize("kind", ["affnet", "orinet", "hardnet"])
def test_simt_ragged_rows(L, kind):
    """A ragged batch through net_forward_rows: groups of 11 rows with counts 11, 0, 5, 1 over a NaN-filled workspace; valid rows carry the
    full batch's bits, the others keep the sentinel."""
    net = module(L, kind, state_dict(kind, "shipped"))
    P = all_patches()[-44:].contiguous()           # the tail: seeded noise and the normalisation's edges
    counts, group = [11, 0, 5, 1], 11
    full, fang = net_forward_rows(L, net, P)
    out, ang = net_forward_rows(L, net, P, counts=counts, group=group, ws_word=0x7FFF)
    valid = torch.tensor([(i % group) < counts[i // group] for i in range(P.size(0))], device=DEV)
    assert bits(out[valid], full[valid]) and (out[~valid] == SENTINEL).all()
    if ang is not None:
        assert bits(ang[valid], fang[valid]) and (ang[~valid] == SENTINEL).all()
