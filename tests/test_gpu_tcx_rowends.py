"""GPU tests of the x neighbours at the ends of image rows in the second-generation tensor-core engine (tcx_first.cuh / tcx_conv.cuh).

The engine stores each 16-slot row group of its activations even-x first, then odd-x, and its epilogues add a pixel's left and right
neighbours from the thread's own values, from lane - 4 / lane + 4, or (32-pixel rows) from the other warp of the row, and drop the
neighbours outside the row by selects.  Patches with bright vertical stripes at input columns 0, 1, 30 and 31 (and 15, 16, where the
first kernel's 32-pixel rows change warp) and constant patches put the largest values right at those row ends; an odd n leaves the
last pair unit's second patch skipped over a NaN-filled workspace, so a padding or neighbour that reaches across a pair's row end
shows up as a wrong or NaN border pixel of the valid patch."""
import pytest
import torch

import affnet_oracle as O
from helpers import gold, load_weights
from test_gpu_tcx import oracle_layers

pytestmark = pytest.mark.gpu
DEV = "cuda"
W = load_weights()
KINDS = ("affnet", "orinet", "hardnet")


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


def rowend_patches():
    """Odd count: bright stripes on seeded noise (one edge column per patch, both edges, the half-row boundary, all four edge columns),
    constant patches and a few graf patches."""
    g = torch.Generator().manual_seed(31)
    P = []
    for cols in ((0,), (1,), (30,), (31,), (0, 31), (15,), (16,), (0, 1, 30, 31)):
        q = torch.rand(1, 1, 32, 32, generator=g) * 40
        q[..., list(cols)] += 200.0
        P.append(q)
    P += [torch.full((1, 1, 32, 32), 77.0), torch.full((1, 1, 32, 32), 0.25)]
    P.append(torch.from_numpy(gold("graf_crop.npz")["aff_patches"])[:9])
    P = torch.cat(P)
    assert P.size(0) % 2 == 1
    return P


@pytest.mark.parametrize("kind", KINDS)
def test_tcx_layers_row_ends_vs_oracle(L, kind):
    """Layers 2..5 decoded from the engine's HBM layouts (ag_debug_tcx_layer) against the fp32 oracle at test_gpu_tcx.py's tolerances
    (relative to the layer's largest activation), for n = all patches, 1 and 3, over a workspace of 0xFF bytes (NaN in fp16)."""
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    net = {"affnet": lambda: AffNetFast(PS=32), "orinet": lambda: OriNetFast(PS=32), "hardnet": HardNet}[kind]()
    net.load_state_dict(W[kind])
    net = net.eval().to(DEV)
    net.set_engine(L.ENGINE_TC2)
    cfg = O.HARDNET_CFG if kind == "hardnet" else O.AFFNET_CFG
    tol = 2e-3 if kind == "hardnet" else 2e-5
    lib = L.lib()
    P_all = rowend_patches()
    for n in (P_all.size(0), 1, 3):
        P = P_all[:n].contiguous()
        ref = oracle_layers(P, W[kind], cfg)
        ws_bytes = lib.ag_net_workspace_bytes(net.KIND, n)
        Pd = P.to(DEV)
        for upto in (2, 3, 4, 5):
            ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device=DEV)
            r = ref[upto - 1]
            out = torch.full(r.shape, float("nan"), device=DEV)
            L.check(lib.ag_debug_tcx_layer(net.handle(), L.ptr(Pd), n, upto, L.ptr(out), L.ptr(ws), ws_bytes, L.stream_ptr()))
            torch.cuda.synchronize()
            o = out.cpu()
            assert not torch.isnan(o).any(), (kind, n, upto)
            rel = (o - r).abs().max().item() / r.abs().max().item()
            # the row ends on their own: first and last column of every map
            rel_ends = (o - r)[..., [0, -1]].abs().max().item() / r.abs().max().item()
            print("\n%s n=%d layer %d: rel %.2e, row ends %.2e" % (kind, n, upto, rel, rel_ends))
            assert rel < tol, (kind, n, upto, rel)


def test_tcx_nets_row_ends_vs_oracle(L):
    """The three nets end to end (layer 6 and the heads included) on the same patches, at test_gpu_tcx.py's tolerances; HardNet's
    descriptors of the constant patches (bias-only activations in single fp16 planes) at test_gpu_rows.py's 2e-3 for flat patches."""
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    a, o, h = a.eval().to(DEV), o.eval().to(DEV), h.eval().to(DEV)
    for m in (a, o, h):
        m.set_engine(L.ENGINE_TC2)
    P = rowend_patches()
    Pd = P.to(DEV)
    dA = (a(Pd).cpu() - O.affnet_forward(P, W["affnet"])).abs().max().item()
    dang = o(Pd, return_rot_matrix=False).cpu() - O.orinet_angle(P, W["orinet"])
    dang = torch.atan2(torch.sin(dang), torch.cos(dang)).abs().max().item()
    eD = (h(Pd).cpu() - O.hardnet_forward(P, W["hardnet"])).abs().amax(1)
    flat = P.reshape(P.size(0), -1).amax(1) == P.reshape(P.size(0), -1).amin(1)
    dD, dD_flat = eD[~flat].max().item(), eD[flat].max().item()
    print("\nrow-end patches: max|dA| %.2e  max|dangle| %.2e rad  max|ddesc| %.2e (flat %.2e)" % (dA, dang, dD, dD_flat))
    assert dA < 5e-5 and dang < 1e-4 and dD < 6e-4 and dD_flat < 2e-3, (dA, dang, dD, dD_flat)
