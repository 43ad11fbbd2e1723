"""CPU tests of the exact-fp32 SIMT engine's restatement (tests/nets_simt_restated.py): it agrees with the oracle and the reference's
goldens, every stage lies within its float64 bound, its cases reach the input normalisation's edges, and each deliberate defect of the
restatement changes bits on those cases, so the GPU test's bit-for-bit comparison would see it in the engine."""
import functools

import numpy as np
import pytest
import torch

import affnet_oracle as O
import nets_simt_restated as S
from helpers import gold, load_weights

W = load_weights()
N_NATURAL = 3


def cases(kind):
    """A few of the graf crop's patches for this net (their golden outputs exist) and the normalisation's edges."""
    z = gold("graf_crop.npz")
    key = {"affnet": "aff_patches", "orinet": "ori_patches", "hardnet": "ori_desc_patches"}[kind]
    return torch.cat([torch.from_numpy(z[key])[:N_NATURAL], S.special_patches()]).contiguous()


@functools.lru_cache(maxsize=None)
def restated(kind, mut=()):
    return S.forward32(cases(kind), W[kind], kind, mut=mut)


def outputs(kind):
    return {"affnet": ("A",), "orinet": ("angle", "R"), "hardnet": ("desc",)}[kind]


def observed(kind):
    """The outputs and the raw head values (AffNet (a00, a10, a11), OriNet (m0, m1)): an unfused head moves the sums by an ulp or two,
    which tanhf and the rectification often absorb on a handful of patches."""
    return outputs(kind) + (("raw",) if kind != "hardnet" else ())


@pytest.mark.parametrize("kind", ["affnet", "orinet", "hardnet"])
def test_restated_within_bounds_and_goldens(kind):
    """Every stage within its float64 bound; the outputs on the graf crop's patches against the reference's goldens and the fp32 oracle."""
    r = restated(kind)
    P = cases(kind)
    outs = {k: r[k] for k in outputs(kind)}
    print()
    S.check_bounds(kind, kind, W[kind], P, r["layers"], outs, r)
    z = gold("graf_crop.npz")
    Pn = P[:N_NATURAL]
    if kind == "affnet":
        got, golden, oracle = r["A"][:N_NATURAL], z["aff_A"][:N_NATURAL], O.affnet_forward(Pn, W[kind])
    elif kind == "orinet":
        got, golden, oracle = r["R"][:N_NATURAL], z["ori_R"][:N_NATURAL], O.orinet_forward(Pn, W[kind])
    else:
        got, golden, oracle = r["desc"][:N_NATURAL], z["ori_desc"][:N_NATURAL], O.hardnet_forward(Pn, W[kind])
    eg = (got - torch.from_numpy(golden).double().reshape(got.shape)).abs().max().item()
    eo = (got - oracle.double().reshape(got.shape)).abs().max().item()
    print("%s: restated vs golden %.2e, vs oracle %.2e" % (kind, eg, eo))
    assert eg < 2e-6 and eo < 2e-6


def test_cases_reach_the_normalisation_edges():
    """Zero and constant patches: q = 0, inv = 1 / 1e-7f.  2^60: q = inf, inv = 0, the staged input all zero.  2^-70: subnormal d * d and
    partial sums of q.  2^-120: every d nonzero but q = 0.  NaN / +-inf pixels: NaN staged inputs, and layer 1's ReLU turns them into 0."""
    r = restated("affnet")
    mean, q, inv = (t[N_NATURAL:] for t in r["stats"])
    xn = r["xn"][N_NATURAL:]
    k = {name: i for i, name in enumerate(S.SPECIAL)}
    big = float(np.float32(1) / np.float32(1e-7))
    for name in ("zero", "constant"):
        assert q[k[name]] == 0 and inv[k[name]] == big and (xn[k[name]] == 0).all()
    assert q[k["times 2^60"]] == float("inf") and inv[k["times 2^60"]] == 0 and (xn[k["times 2^60"]] == 0).all()
    P = cases("affnet")[N_NATURAL:].double().reshape(-1, 32, 32)
    d = S.r32(P - mean.view(-1, 1, 1))
    dd = S.fma(d, d, torch.zeros_like(d))
    i = k["times 2^-70"]
    sub = (dd[i] > 0) & (dd[i] < 2.0 ** -126)
    assert sub.any() and (dd[i] >= 2.0 ** -126).any() and 0 < q[i] < 2.0 ** -100
    i = k["times 2^-120"]
    assert (d[i] != 0).all() and q[i] == 0 and inv[i] == big and (xn[i] != 0).all()
    for name in ("NaN pixel", "+inf pixel", "-inf pixel"):
        assert torch.isnan(xn[k[name]]).all()
        assert (r["layers"][0][N_NATURAL + k[name]] == 0).all() and torch.isfinite(r["A"][N_NATURAL + k[name]]).all()
    assert torch.isinf(mean[k["+inf pixel"]]) and torch.isinf(mean[k["-inf pixel"]]) and torch.isnan(mean[k["NaN pixel"]])


MUTATION_NET = {"tap_major": "affnet", "contiguous_head": "orinet", "pairwise_reduce": "hardnet", "norm_distributed": "affnet",
                "unfused_affnet_head": "affnet", "hardnet_shift_invstd": "hardnet", "pad_shift_row_end": "affnet"}


@pytest.mark.parametrize("mutation", S.MUTATIONS)
def test_mutations_change_bits(mutation):
    """Each deliberate defect changes the bits of the outputs or of the raw head values on the cases."""
    kind = MUTATION_NET[mutation]
    base, mut = restated(kind), restated(kind, (mutation,))
    changed = {k: int((base[k].float().view(torch.int32) != mut[k].float().view(torch.int32)).any(dim=tuple(range(1, base[k].dim()))).sum())
               for k in observed(kind)}
    print("\n%s on %s: patches with changed outputs %s of %d" % (mutation, kind, changed, cases(kind).size(0)))
    assert any(changed.values()), mutation


def test_mutations_are_named():
    assert set(MUTATION_NET) == set(S.MUTATIONS)
