"""GPU tests (-m gpu): the Gaussian blur, the pyramid, the Hessian response and the patch samplers bit for bit against the exact fp32
restatement of their arithmetic (tests/scale_space_restated.py, run in float64 on the device), and within derived bounds of the
reference's float64 operations.  Outputs are prefilled with a sentinel so that a missing or stray write is seen.  Which blur fill and
store paths these cases reach is asserted on the CPU (tests/test_scale_space_cpu.py)."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import affnet_oracle as O
import scale_space_cases as K
import scale_space_restated as R
from helpers import gold, gray_from_rgb

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = -777.25
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


def bits_equal(a, b):
    a, b = a.to(torch.float32).contiguous(), b.to(a.device, torch.float32).contiguous()
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def ndiff(a, b):
    return int((a.to(torch.float32).contiguous().view(torch.int32) != b.to(a.device, torch.float32).contiguous().view(torch.int32)).sum())


def noise(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(*shape, generator=g) * 255).to(DEV)


def fma_separate(a, b, c):
    """The mutation of the restatement: round(round(a*b) + c) instead of the fused multiply-add."""
    return R._f32(R._t64(R._f32(R._t64(a) * R._t64(b))) + R._t64(c))


def blur(L, x, out, B, h, w, sigma):
    return L.lib().ag_gaussian_blur(L.ptr(x), L.ptr(out), B, h, w, float(sigma), L.stream_ptr())


# ---- a. ag_gaussian_blur ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", K.BLUR_BATCHES)
def test_blur_bit_exact_every_radius_and_shape(L, B):
    mutant_caught, mutant_cases = 0, 0
    for (h, w) in K.BLUR_SHAPES:
        x = noise((B, h, w), h * 1000 + w + B)
        for r in K.RADII:
            s = K.sigma_for_radius(r)
            out = torch.full((B, h, w), SENT, device=DEV)
            L.check(blur(L, x, out, B, h, w, s))
            ref = R.blur32(x, s)
            assert bits_equal(out, ref), (B, h, w, r, ndiff(out, ref))
            if h * w >= 15:
                mutant_cases += 1
                mutant_caught += not bits_equal(out, R.blur32(x, s, descending=True))
    # the check is sharp: summing the taps in descending order is seen (all but a few tiny images have some pixel that differs)
    print("\nB %d: the descending-order restatement disagrees in %d of %d cases" % (B, mutant_caught, mutant_cases))
    assert mutant_caught >= 0.9 * mutant_cases


def test_blur_misaligned_pointers(L):
    """Input and output 1-3 floats past a 16-byte boundary: the scalar fill and scalar stores, same bits, nothing written outside."""
    for (h, w) in K.OFFSET_SHAPES:
        for B in K.BLUR_BATCHES:
            n = B * h * w
            x = noise((n,), h + w + B)
            for r in K.OFFSET_RADII:
                s = K.sigma_for_radius(r)
                ref = R.blur32(x.view(B, h, w), s).reshape(-1)
                for io, oo in K.OFFSETS:
                    src = torch.full((n + 8,), SENT, device=DEV)
                    src[io:io + n] = x
                    dst = torch.full((n + 8,), SENT, device=DEV)
                    rc = L.lib().ag_gaussian_blur(C.c_void_p(src.data_ptr() + 4 * io), C.c_void_p(dst.data_ptr() + 4 * oo), B, h, w, float(s),
                                                  L.stream_ptr())
                    L.check(rc)
                    assert bits_equal(dst[oo:oo + n], ref), (h, w, B, r, io, oo, ndiff(dst[oo:oo + n], ref))
                    assert bool((dst[:oo] == SENT).all()) and bool((dst[oo + n:] == SENT).all()), (h, w, B, r, io, oo)


def test_blur_refuses_radius_13(L):
    x = noise((1, 40, 40), 1)
    out = torch.full_like(x, SENT)
    rc = blur(L, x, out, 1, 40, 40, 4.25)
    assert rc != 0
    assert L.lib().ag_last_error().decode() == "gaussian sigma 4.2500 needs 27 taps (max 25)"
    torch.cuda.synchronize()
    assert bool((out == SENT).all())


# ---- b/d. ag_pyramid_build --------------------------------------------------------------------------------------------------------
def case_input(case):
    name, B, H, W = case[:4]
    if name == "graf":
        return gray_from_rgb(gold("graf_crop.npz")["rgb"]).view(1, H, W).to(DEV)
    return noise((B, H, W), B * 7919 + H * 31 + W)


def build(L, plan, x):
    buf = torch.full((plan.total_floats,), SENT, device=DEV)
    rc = L.lib().ag_pyramid_build(C.byref(plan), L.ptr(x), L.ptr(buf), L.stream_ptr())
    return rc, buf


def level(plan, buf, o, l):
    n = plan.B * plan.h[o] * plan.w[o]
    off = plan.level_offset[o][l]
    return buf[off:off + n].view(plan.B, plan.h[o], plan.w[o])


def needs_too_many_taps(plan):
    return [O.gauss_kernel_size(sig) for _, _, sig, _, _ in K.pyramid_blurs(plan) if O.gauss_kernel_size(sig) > K.MAX_TAPS]


def check_pyramid(plan, buf, x, tag):
    pyr = R.pyramid32(x, plan)
    for o in range(plan.n_octaves):
        for l in range(plan.n_levels):
            got = level(plan, buf, o, l)
            assert bits_equal(got, pyr[o][l]), (tag, o, l, ndiff(got, pyr[o][l]))
    return pyr


def float64_contract(plan, buf, x, tag):
    """Every level within the summed one-blur bounds of the float64 chain of the reference's dense blurs; returns the worst ratio."""
    p64 = R.pyramid64(x, plan)
    bounds = R.pyramid_bounds(plan)
    m = x.abs().max().item()
    worst = (0.0, 0.0, 0.0)
    for o in range(plan.n_octaves):
        for l in range(plan.n_levels):
            err = (level(plan, buf, o, l).double() - p64[o][l]).abs().max().item()
            bound = bounds[o][l] * m
            assert err <= bound, (tag, o, l, err, bound)
            if bound > 0 and err / bound > worst[0]:
                worst = (err / bound, err, bound)
    return worst


@pytest.mark.parametrize("case", K.PYR_CASES, ids=lambda c: "%s-B%d-%dx%d-nl%d-s%g-b%d" % c)
def test_pyramid_bit_exact(L, case):
    _, B, H, W, nl, s, border = case
    plan = L.make_plan(B, H, W, nl, s, border)
    x = case_input(case)
    rc, buf = build(L, plan, x)
    too_many = needs_too_many_taps(plan)
    if too_many:
        assert rc != 0
        assert re.fullmatch(r"gaussian sigma \d+\.\d{4} needs %d taps \(max 25\)" % too_many[0], L.lib().ag_last_error().decode())
        torch.cuda.synchronize()
        assert bool((buf == SENT).all()), "a refused pyramid wrote to its buffer"
        return
    L.check(rc)
    check_pyramid(plan, buf, x, case)
    if s <= 0.5:
        assert plan.blur_sigma[0][0] == 0.0 and bits_equal(level(plan, buf, 0, 0), x)
    worst = float64_contract(plan, buf, x, case)
    print("\n%s: %d octaves, worst float64 error %.3g = %.3f of its bound %.3g; misaligned levels %s"
          % (case, plan.n_octaves, worst[1], worst[0], worst[2], K.misaligned_levels(plan)))
    if (B, H, W, nl, s) == (1, 97, 127, 3, 1.6):
        # the mutation check: the restatement with the taps summed in descending order disagrees
        pyr_m = R.pyramid32(x, plan, descending=True)
        assert not bits_equal(level(plan, buf, 0, 2), pyr_m[0][2])


def test_pyramid_nlevels_1_refused(L):
    plan = L.make_plan(1, 97, 127, 1, 1.6, 5)
    rc, buf = build(L, plan, noise((1, 97, 127), 3))
    assert rc != 0 and L.lib().ag_last_error().decode() == "gaussian sigma 5.5426 needs 35 taps (max 25)"
    torch.cuda.synchronize()
    assert bool((buf == SENT).all())


def test_pyramid_batch_equals_single_images(L):
    B, H, W, nl, s, border = K.BATCH_CASE
    x = noise((B, H, W), 99)
    plan = L.make_plan(B, H, W, nl, s, border)
    rc, buf = build(L, plan, x)
    L.check(rc)
    check_pyramid(plan, buf, x, "batch")
    for b in range(B):
        p1 = L.make_plan(1, H, W, nl, s, border)
        rc, b1 = build(L, p1, x[b:b + 1].contiguous())
        L.check(rc)
        for o in range(plan.n_octaves):
            for l in range(plan.n_levels):
                assert bits_equal(level(plan, buf, o, l)[b], level(p1, b1, o, l)[0]), (b, o, l)


_NO_TMA = r"""
import ctypes as C, sys, torch
for p in ("", "/oracle", "/tests"):
    sys.path.insert(0, sys.argv[2] + p)
import affnet_b200._lib as L
import scale_space_cases as K
from test_gpu_scale_space import case_input, build, noise, blur, SENT
L.lib()
out = {}
for case in K.NO_TMA_PYR_CASES:
    plan = L.make_plan(*case[1:])
    rc, buf = build(L, plan, case_input(case))
    L.check(rc)
    out[str(case)] = buf.cpu()
for B, h, w, r in K.NO_TMA_BLUR_CASES:
    x = noise((B, h, w), 5)
    o = torch.full_like(x, SENT)
    L.check(blur(L, x, o, B, h, w, K.sigma_for_radius(r)))
    out[str((B, h, w, r))] = o.cpu()
torch.save(out, sys.argv[1])
"""


def test_pyramid_without_tensor_maps_bit_exact(L, tmp_path):
    """AG_BLUR_NO_TMA=1 (a driver without the tensor-map encoder): interior tiles take per-row bulk copies."""
    path = str(tmp_path / "no_tma.pt")
    env = dict(os.environ)
    env["AG_BLUR_NO_TMA"] = "1"
    r = subprocess.run([sys.executable, "-c", _NO_TMA, path, ROOT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    got = torch.load(path)
    for case in K.NO_TMA_PYR_CASES:
        plan = L.make_plan(*case[1:])
        check_pyramid(plan, got[str(case)].to(DEV), case_input(case), ("no tma",) + case)
    for B, h, w, r in K.NO_TMA_BLUR_CASES:
        assert bits_equal(got[str((B, h, w, r))].to(DEV), R.blur32(noise((B, h, w), 5), K.sigma_for_radius(r))), (B, h, w, r)


# ---- c. ag_hessian_response -------------------------------------------------------------------------------------------------------
def test_hessian_bit_exact_batched_odd_shapes(L):
    for (h, w) in K.BLUR_SHAPES:
        x = O.gaussian_blur(noise((3, 1, h, w), h + 3 * w).cpu(), 1.2)
        for s in (1.6, 2.0158736798317967):
            ref = O.hessian_response(x, s)
            for th in (0.0, 5.0):
                out = torch.full((3, 1, h, w), SENT, device=DEV)
                L.check(L.lib().ag_hessian_response(L.ptr(x.to(DEV)), L.ptr(out), 3, h, w, float(s), float(th), L.stream_ptr()))
                exp = torch.clamp(ref - th, min=0.0) if th > 0 else ref
                assert bits_equal(out, exp), (h, w, s, th, ndiff(out, exp))


# ---- e. ag_extract_patches ----------------------------------------------------------------------------------------------------------
IMG_H, IMG_W = 64, 128          # min(h, w) and w are powers of two: the axis-aligned LAFs below are exact in fp32


def laf_sets(n_rand, seed):
    g = torch.Generator().manual_seed(seed)
    sets = {}
    A = (torch.rand(n_rand, 2, 2, generator=g) - 0.5) * 0.8
    t = torch.rand(n_rand, 2, 1, generator=g) * 1.4 - 0.2
    sets["random"] = torch.cat([A, t], 2)
    rows = []
    for PSs in (1, 2, 8, 32):             # sample spacing of 1 and 2 pixels for these patch sizes; centres on pixel centres and edges
        for sp in (1.0, 2.0):
            a = PSs / 2.0 * sp / min(IMG_H, IMG_W)
            for cx, cy in ((40.5, 20.5), (41.0, 21.0), (0.5, 0.5), (127.5, 63.0)):
                rows.append([[a, 0.0, cx / IMG_W], [0.0, a, cy / IMG_H]])
    sets["axis"] = torch.tensor(rows)
    rows = []
    for cx, cy in ((-1.0, 0.5), (2.0, 0.5), (0.5, -1.0), (0.5, 2.0)):      # wholly outside
        rows.append([[0.1, 0.0, cx], [0.0, 0.1, cy]])
    for cx, cy in ((0.0, 0.5), (1.0, 0.5), (0.5, 0.0), (0.5, 1.0)):        # partly outside, across each edge
        rows.append([[0.1, 0.03, cx], [-0.02, 0.1, cy]])
    rows.append([[0.0, 0.0, 0.3], [0.0, 0.0, 0.6]])                        # A = 0
    rows.append([[0.0, 0.0, 0.3], [0.0, 0.0, 0.0]])
    for sc in (30.0, 1e4, 1e8):                                           # very large scales, up to past the int32 range of floorf
        rows.append([[sc, 0.3 * sc, 0.5], [-0.2 * sc, sc, 0.5]])
    sets["edges"] = torch.tensor(rows)
    return sets


@pytest.mark.parametrize("PS", [1, 2, 19, 32, 41, 64])
@pytest.mark.parametrize("Cc", [1, 3])
@pytest.mark.parametrize("per_patch", [0, 1])
def test_extract_patches_bit_exact(L, PS, Cc, per_patch):
    worst = (0.0, 0.0, 0.0)
    caught = 0
    for name, lafs in laf_sets(24, PS * 10 + Cc).items():
        n = lafs.size(0)
        lafs = lafs.float().to(DEV).contiguous()
        m = n if per_patch else 1
        img = noise((m, Cc, IMG_H, IMG_W), PS + Cc + per_patch + n)
        out = torch.full((n, Cc, PS, PS), SENT, device=DEV)
        L.check(L.lib().ag_extract_patches(L.ptr(img), Cc, IMG_H, IMG_W, per_patch, L.ptr(lafs), n, PS, L.ptr(out), L.stream_ptr()))
        sel = torch.arange(n) if per_patch else None
        for c in range(Cc):
            ref = R.sample32(img[:, c], lafs, PS, sel)
            assert bits_equal(out[:, c], ref), (name, PS, Cc, per_patch, c, ndiff(out[:, c], ref))
            caught += not bits_equal(out[:, c], R.sample32(img[:, c], lafs, PS, sel, fma=fma_separate))
        if name != "edges" and not per_patch:
            for c in range(Cc):
                e = (out[:, c].double().cpu() - R.sample64(img[0, c].cpu(), lafs.cpu(), PS)).abs().max().item()
                bd = R.sample_bound(img[0, c].cpu(), lafs.cpu())
                assert e <= bd, (name, PS, c, e, bd)
                worst = max(worst, (e / bd, e, bd))
    # the check is sharp: a separate multiply and add instead of the FMA is seen
    assert caught > 0
    if not per_patch:
        print("\nPS %d C %d: sampler vs float64 %.3g = %.3f of its bound %.3g" % (PS, Cc, worst[1], worst[0], worst[2]))


def test_extract_patches_counts(L):
    lib = L.lib()
    img = noise((1, 1, 40, 50), 2)
    lafs = torch.zeros(65536, 2, 3, device=DEV)
    lafs[:, 0, 0] = 0.1; lafs[:, 1, 1] = 0.1; lafs[:, :, 2] = 0.5
    out = torch.full((4,), SENT, device=DEV)
    L.check(lib.ag_extract_patches(L.ptr(img), 1, 40, 50, 0, L.ptr(lafs), 0, 2, L.ptr(out), L.stream_ptr()))       # n = 0
    torch.cuda.synchronize()
    assert bool((out == SENT).all())
    big = torch.full((65536, 1, 2, 2), SENT, device=DEV)
    assert lib.ag_extract_patches(L.ptr(img), 1, 40, 50, 0, L.ptr(lafs), 65536, 2, L.ptr(big), L.stream_ptr()) != 0
    assert lib.ag_last_error().decode() == "ag_extract_patches: n too large for one launch (max 65535)"
    torch.cuda.synchronize()
    assert bool((big == SENT).all())
    from affnet_b200.LAF import extract_patches
    g = torch.Generator().manual_seed(8)
    many = torch.cat([(torch.rand(70000, 2, 2, generator=g) - 0.5) * 0.3, torch.rand(70000, 2, 1, generator=g)], 2).to(DEV)
    got = extract_patches(img, many, PS=2)
    assert bits_equal(got[:, 0], R.sample32(img[:, 0], many, 2))


# ---- f. ag_extract_patches_pyr ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("counts", [(0, 3), (7, -1), (5, 7), None], ids=["0-partial", "full-neg", "partial-full", "null"])
def test_extract_patches_pyr_rows_and_clamped_indices(L, counts):
    B, H, W, cap, PS = 2, 97, 127, 7, 19
    plan = L.make_plan(B, H, W, 3, 1.6, 5)
    x = noise((B, H, W), 17)
    rc, buf = build(L, plan, x)
    L.check(rc)
    g = torch.Generator().manual_seed(4)
    lafs = torch.cat([(torch.rand(B, cap, 2, 2, generator=g) - 0.5) * 0.4, torch.rand(B, cap, 2, 1, generator=g)], 3).to(DEV)
    oc = torch.tensor([[0, 1, 2, -3, 99, 1, 0], [2, 0, -1, 1, 7, 0, 1]], dtype=torch.int32, device=DEV)
    lv = torch.tensor([[0, 4, 2, 1, -5, 9, 3], [1, 3, 0, 4, 2, 100, -1]], dtype=torch.int32, device=DEV)
    cnt = None if counts is None else torch.tensor(counts, dtype=torch.int32, device=DEV)
    out = torch.full((B, cap, PS, PS), SENT, device=DEV)
    L.check(L.lib().ag_extract_patches_pyr(C.byref(plan), L.ptr(buf), L.ptr(lafs), L.ptr(oc), L.ptr(lv), L.ptr(cnt), cap, PS, L.ptr(out),
                                           L.stream_ptr()))
    for b in range(B):
        n = cap if counts is None else max(0, min(counts[b], cap))
        for i in range(cap):
            if i >= n:
                assert bool((out[b, i] == SENT).all()), (b, i)
                continue
            o = min(max(int(oc[b, i]), 0), plan.n_octaves - 1)
            l = min(max(int(lv[b, i]), 0), plan.n_levels - 1)
            ref = R.sample32(level(plan, buf, o, l)[b:b + 1], lafs[b, i:i + 1], PS)[0]
            assert bits_equal(out[b, i], ref), (b, i, o, l)


# ---- g. ag_pyramid_level_for_lafs ---------------------------------------------------------------------------------------------------
def test_level_for_lafs_ties_go_to_the_first_candidate(L):
    """nlevels 1, init_sigma 1: the candidates sigma * 2^o are 1 2 4 | 2 4 8 | 4 8 16, exact in float64.  A LAF with scale needed * PS
    (needed exact in fp32) is exactly equidistant from two candidates (or equal to two); numpy's argmin takes the first."""
    from affnet_b200.LAF import get_pyramid_and_level_index_for_LAFs
    PS = 32
    plan = L.make_plan(1, 64, 64, 1, 1.0, 5)
    sig = [[plan.sigma[o][l] for l in range(plan.n_levels)] for o in range(plan.n_octaves)]
    pix = [[plan.pix_dist[o]] * plan.n_levels for o in range(plan.n_octaves)]
    cand, _, _ = O.level_candidates(sig, pix)
    assert list(cand) == [1, 2, 4, 2, 4, 8, 4, 8, 16]
    needed = [0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0, 8.0, 12.0, 16.0, 100.0, 2.5, 0.75]
    lafs = torch.zeros(len(needed), 2, 3)
    for i, v in enumerate(needed):
        lafs[i, 0, 0] = lafs[i, 1, 1] = v * PS
    d = np.abs(cand.reshape(-1, 1) - np.array(needed).reshape(1, -1))
    ties = int(((d == d.min(0, keepdims=True)).sum(0) > 1).sum())
    assert ties == 8                      # 1.5 2 2.5 3 4 6 8 12 (2, 4 and 8 are candidates twice)
    o_ref, l_ref = O.pyramid_level_for_lafs(lafs, sig, pix, PS)
    o, l = get_pyramid_and_level_index_for_LAFs(lafs.to(DEV), plan, PS)
    assert o.cpu().tolist() == o_ref.int().tolist() and l.cpu().tolist() == l_ref.int().tolist()
    # e.g. needed 3 lies between 2 (octave 0, level 1) and 4 (octave 0, level 2): the first candidate, level 1, wins
    assert (o[4].item(), l[4].item()) == (0, 1)
