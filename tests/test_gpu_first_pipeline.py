"""GPU tests (-m gpu) of the pipelined first-layers kernel (tcx_first_kernel: two blocks in flight per consumer warpgroup, P-plane halves
released after layer 1, layer 3 of AffNet / OriNet in the same kernel) at patch counts that reach its prologue and drain paths: a CTA
with one patch, CTAs that get one patch more than others (n = 131, 132, 133 against the 132 SMs of an H100), CTAs with two and more
patches, and device row-count arrays whose groups hold 0, 1, an odd number and all of their rows.

Every valid patch must be bit-identical to the same patch run alone (n = 1), whatever the workspace held (poisoned with NaN or +Inf
words as in test_gpu_rows.py), and rows beyond the counts must keep their sentinel."""
import pytest
import torch

from helpers import POISON_INF, POISON_NAN, SENTINEL, gold, load_weights, net_forward_rows, row_valid

pytestmark = pytest.mark.gpu
DEV = "cuda"
W = load_weights()
# (net, engine): the default engine of each net, and HardNet's bf16 variant (its own tcx_first_kernel instantiation)
CASES = [("affnet", "ENGINE_TC2"), ("orinet", "ENGINE_TC2"), ("hardnet", "ENGINE_TC2"), ("hardnet", "ENGINE_TC2_BF16")]
DENSE_N = (1, 2, 131, 132, 133, 265)
# (n, group, counts): groups with 0, 1, an odd count and the full group; a group size that does not divide n
GROUPED = [(132, 33, [0, 1, 17, 33]), (265, 53, [53, 0, 1, 27, 53]), (133, 19, [1, 19, 0, 7, 19, 3, 11])]


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


@pytest.fixture(scope="module")
def nets(L):
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    return {"affnet": a.eval().to(DEV), "orinet": o.eval().to(DEV), "hardnet": h.eval().to(DEV)}


@pytest.fixture(scope="module")
def pool():
    """101 distinct patches: graf-crop patches, seeded uniform patches in [0, 255) and [0, 1), a constant one."""
    z = gold("graf_crop.npz")
    g = torch.Generator().manual_seed(21)
    P = torch.cat([torch.from_numpy(z["aff_patches"])[:60], torch.rand(20, 1, 32, 32, generator=g) * 255,
                   torch.rand(20, 1, 32, 32, generator=g), torch.full((1, 1, 32, 32), 77.0)])
    return P[torch.randperm(P.size(0), generator=torch.Generator().manual_seed(22))]


def bits(t):
    return t.contiguous().view(torch.int32).reshape(t.size(0), -1)


@pytest.mark.parametrize("kind,engine", CASES, ids=["%s-%s" % (k, e[7:].lower()) for k, e in CASES])
def test_first_kernel_edges_bit_identical_to_single_patches(L, nets, pool, kind, engine):
    net = nets[kind]
    N = pool.size(0)
    sentinel = bits(torch.tensor([SENTINEL]))[0, 0].item()
    net.set_engine(getattr(L, engine))
    try:
        # every pool patch alone: one CTA, one patch (prologue and drain of the same patch)
        single = []
        for i in range(N):
            out, angle = net_forward_rows(L, net, pool[i:i + 1].to(DEV), None, 0, ws_word=POISON_NAN)
            single.append(torch.cat([bits(out.cpu())] + ([bits(angle.cpu())] if angle is not None else []), 1))
        single = torch.cat(single)
        failures = []
        runs = [(n, n, None) for n in DENSE_N] + GROUPED
        for n, group, counts in runs:
            idx = torch.arange(n) % N
            valid = row_valid(n, group, counts)
            for word in (POISON_NAN, POISON_INF):
                tag = "n=%d group=%d counts=%s poison=0x%04X" % (n, group, counts, word)
                out, angle = net_forward_rows(L, net, pool[idx].to(DEV), counts, group, ws_word=word)
                got = torch.cat([bits(out.cpu())] + ([bits(angle.cpu())] if angle is not None else []), 1)
                vi = valid.nonzero().view(-1)
                diff = (got[vi] != single[idx[vi]]).any(1)
                if diff.any():
                    failures.append("%s: valid rows differ from the patch run alone: %s" % (tag, vi[diff][:12].tolist()))
                inv = got[~valid]
                if inv.numel() and not bool((inv == sentinel).all()):
                    rows = (~valid).nonzero().view(-1)[(inv != sentinel).any(1)]
                    failures.append("%s: rows beyond the counts written: %s" % (tag, rows[:12].tolist()))
    finally:
        net.set_engine(L.ENGINE_TC2)
    assert not failures, "\n".join(failures[:40])
