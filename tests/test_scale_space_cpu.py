"""CPU tests of the fp32 restatement of the blur, pyramid and sampler (tests/scale_space_restated.py) that the GPU tests hold the kernels
to bit for bit, and of the coverage of those GPU cases: every input fill path and output store path of blur_kernel, every radius, and
pyramid levels that start off a 16-byte boundary."""
import collections
import ctypes

import numpy as np
import pytest
import torch

import affnet_oracle as O
import scale_space_cases as K
import scale_space_restated as R

libm = ctypes.CDLL("libm.so.6")
libm.fmaf.restype = ctypes.c_float
libm.fmaf.argtypes = [ctypes.c_float] * 3


def _glibc_fmaf(a, b, c):
    return np.array([libm.fmaf(float(x), float(y), float(z)) for x, y, z in zip(a, b, c)], np.float32)


def _bits(x):
    return np.asarray(x, np.float32).view(np.int32)


def test_fmaf32_equals_glibc_fmaf_on_random_triples():
    rng = np.random.default_rng(0)
    n = 40000
    sets = [
        (rng.standard_normal(n), rng.random(n) * 0.3, rng.random(n) * 255),                 # blur taps times pixels plus an accumulator
        (rng.standard_normal(n) * 1e3, rng.standard_normal(n) * 1e-3, rng.standard_normal(n)),
        (rng.standard_normal(n), rng.standard_normal(n), -rng.random(n) * 1e-6),            # cancellation-free tiny addends
    ]
    total = 0
    for a, b, c in sets:
        a, b, c = (v.astype(np.float32) for v in (a, b, c))
        assert np.array_equal(_bits(R.fmaf32(a, b, c)), _bits(_glibc_fmaf(a, b, c)))
        total += n
    # products that cancel against the addend: the exact result is far below the operands' ulps
    a = rng.standard_normal(n).astype(np.float32)
    b = rng.standard_normal(n).astype(np.float32)
    c = (-(a.astype(np.float64) * b.astype(np.float64))).astype(np.float32)
    assert np.array_equal(_bits(R.fmaf32(a, b, c)), _bits(_glibc_fmaf(a, b, c)))
    total += n
    assert total >= 100000


def test_fmaf32_breaks_exact_midpoints_by_the_twosum_tail():
    """Triples whose float64 sum s = fl64(a*b + c) lies exactly on an fp32 midpoint while a*b + c does not: rounding s alone ties to
    even, the correct result goes to the side of the tail e.  With c = (1 + m 2^-23) 2^q and a*b = h 2^q (1 + d), h an odd multiple of
    2^-24 (so c + h 2^q is a midpoint) and 0 < |d| < 2^-31 (so the float64 sum drops d), the tie is decided by d alone:
      d < 0: a = h 2^q (1 + i 2^-23), b = 1 - i 2^-23, d = -i^2 2^-46;
      d > 0: a = h 2^q (1 + 2^-k),   b = fp32(1 / (1 + 2^-k)), d = the rounding of b (it leaves a*b just above or below h 2^q)."""
    a, b, c = [], [], []
    for q in (-20, 0, 20):
        for hm in (1, 3, 5, 7):
            h = hm * 2.0 ** -24 * 2.0 ** q
            for m in range(8):
                cc = (1.0 + m * 2.0 ** -23) * 2.0 ** q
                for sign in (1.0, -1.0):
                    for i in range(1, 65):
                        a.append(sign * h * (1.0 + i * 2.0 ** -23)); b.append(1.0 - i * 2.0 ** -23); c.append(sign * cc)
                    for k in range(8, 24):
                        a.append(sign * h * (1.0 + 2.0 ** -k)); b.append(float(np.float32(1.0 / (1.0 + 2.0 ** -k)))); c.append(sign * cc)
    a, b, c = (np.array(v, np.float64).astype(np.float32) for v in (a, b, c))
    ref = _glibc_fmaf(a, b, c)
    assert np.array_equal(_bits(R.fmaf32(a, b, c)), _bits(ref))
    # the triples where rounding the float64 sum alone is wrong: the tail decided them
    naive = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)
    wrong = int((_bits(naive) != _bits(ref)).sum())
    print("\n%d constructed midpoint triples, %d of them rounded wrongly from the float64 sum alone" % (len(a), wrong))
    assert wrong >= 1000


@pytest.mark.parametrize("radius", K.RADII)
def test_taps_equal_the_reference_factor_rounded_to_fp32(radius):
    s = K.sigma_for_radius(radius)
    t = R.taps(s)
    assert len(t) == 2 * radius + 1
    assert np.array_equal(_bits(t), _bits(O.gauss_kernel_1d(s).astype(np.float32)))


def test_blur32_within_the_float64_bound():
    g = torch.Generator().manual_seed(5)
    worst = 0.0
    for (h, w) in ((37, 43), (9, 1), (64, 70)):
        x = torch.rand(2, h, w, generator=g) * 255
        for radius in (1, 5, 12):
            s = K.sigma_for_radius(radius)
            err = (R.blur32(x, s).double() - R.blur64(x, s)).abs().max().item()
            bound = R.blur_bound(s) * x.abs().max().item()
            worst = max(worst, err / bound)
            assert err <= bound, (h, w, radius, err, bound)
    print("\nblur32 vs the float64 dense blur: worst error / bound = %.3f" % worst)


def test_sample32_within_the_float64_bound():
    g = torch.Generator().manual_seed(6)
    img = torch.rand(1, 41, 57, generator=g) * 255
    lafs = torch.cat([(torch.rand(64, 2, 2, generator=g) - 0.5) * 0.6, torch.rand(64, 2, 1, generator=g) * 1.4 - 0.2], 2)
    err = (R.sample32(img, lafs, 19).double() - R.sample64(img, lafs, 19)).abs().max().item()
    bound = R.sample_bound(img[0], lafs)
    print("\nsample32 vs the float64 sampler: %.3g (bound %.3g)" % (err, bound))
    assert err <= bound


def _plan(B, H, W, nl, s, border):
    import affnet_b200._lib as L
    return L.make_plan(B, H, W, nl, s, border)


def _needs_too_many_taps(plan):
    return any(O.gauss_kernel_size(sig) > K.MAX_TAPS for h, w, sig, _, _ in K.pyramid_blurs(plan))


def test_gpu_cases_reach_every_fill_and_store_path_and_radius():
    """Classify every CTA of every blur the GPU file launches, as blur_kernel picks its paths.  A case list that silently stopped
    reaching a path would leave that path untested."""
    paths, radii = collections.Counter(), set()
    for (h, w) in K.BLUR_SHAPES:
        for B in K.BLUR_BATCHES:
            for r in K.RADII:
                paths += K.blur_tile_paths(B, h, w, r)
                radii.add(r)
    for (h, w) in K.OFFSET_SHAPES:
        for B in K.BLUR_BATCHES:
            for r in K.OFFSET_RADII:
                for io, oo in K.OFFSETS:
                    paths += K.blur_tile_paths(B, h, w, r, io, oo)
    for B, h, w, r in K.NO_TMA_BLUR_CASES:
        paths += K.blur_tile_paths(B, h, w, r, tma=False)
    misaligned = []
    for case in K.PYR_CASES + [("noise",) + K.BATCH_CASE]:
        _, B, H, W, nl, s, border = case
        plan = _plan(B, H, W, nl, s, border)
        if _needs_too_many_taps(plan):
            continue
        for h, w, sig, io, oo in K.pyramid_blurs(plan):
            r = R.radius(sig)
            radii.add(r)
            paths += K.blur_tile_paths(B, h, w, r, io or 0, oo)
        if K.misaligned_levels(plan):
            misaligned.append((case, K.misaligned_levels(plan)))
    for case in K.NO_TMA_PYR_CASES:
        _, B, H, W, nl, s, border = case
        for h, w, sig, io, oo in K.pyramid_blurs(_plan(B, H, W, nl, s, border)):
            paths += K.blur_tile_paths(B, h, w, R.radius(sig), io or 0, oo, tma=False)
    print("\nblur CTAs by path:", dict(paths))
    print("pyramid cases with a misaligned level of width % 4 == 0:", len(misaligned))
    for case, lv in misaligned[:6]:
        print("   ", case, lv)
    for p in ("tma", "bulk", "ldg128", "scalar", "store_v4", "store_scalar"):
        assert paths[p] > 0, p
    assert radii == set(K.RADII)
    assert len(misaligned) >= 3
    shapes = {(c[1], c[2], c[3]) for c, _ in misaligned}
    assert {(1, 97, 127), (2, 97, 127), (1, 767, 1023)} <= shapes, shapes


def test_refused_pyramid_cases_are_the_ones_that_need_more_than_25_taps():
    refused = [c for c in K.PYR_CASES if _needs_too_many_taps(_plan(*c[1:]))]
    assert refused == [("noise", 1, 97, 127, 1, 1.6, 5), ("noise", 1, 97, 127, 1, 2.0, 5)], refused
    # nlevels 2 at init_sigma 2.0 needs exactly 25 taps (sigma 4.000000000000002): the largest schedule that runs
    plan = _plan(1, 97, 127, 2, 2.0, 5)
    assert max(O.gauss_kernel_size(sig) for _, _, sig, _, _ in K.pyramid_blurs(plan)) == 25
