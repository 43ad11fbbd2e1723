"""CPU tests of the detector's soft-argmax restatement (tests/detect_restated.py) and of the inputs tests/test_gpu_detect_exact.py
feeds the detector (tests/detect_cases.py): the rounding helpers against numpy and glibc, the oracle and the reference's goldens
within the float64 bound, both kernel orders within it, the cases reaching the soft-argmax's edges, and every listed mutation of
the restatement changing at least one row's bits on those cases."""
import ctypes
import ctypes.util

import numpy as np
import pytest
import torch

import affnet_oracle as O
import detect_cases as DC
from detect_restated import ORDERS, Restated, add, bits, bound_ratio, div, mul
from helpers import OracleCandidates, gold, gray_from_rgb
from scale_space_restated import fmaf32

MR = 5.192
MUTATIONS = ("swap_order", "no_eps", "den_times_min", "split_y", "xy_swap", "scale_first")


def _f32_values(g, n):
    """fp32 values of every kind: normal over a wide exponent range, subnormal, zeros of both signs."""
    e = torch.randint(-149, 40, (n,), generator=g).double()
    m = torch.rand(n, generator=g, dtype=torch.float64) + 1.0
    s = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0).double()
    v = (s * m * torch.pow(2.0, e)).float()
    v[:8] = torch.tensor([0.0, -0.0, 1e-45, -1e-45, 2.0 ** -126, 2.0 ** -127, 3.0 * 2.0 ** -149, 1.0])
    return v


def test_rounding_helpers_against_numpy_and_glibc():
    assert float(torch.tensor(2.0 ** -140, dtype=torch.float32) * 0.5) != 0.0, "torch flushes subnormals: restatement invalid"
    assert float(torch.tensor([2.0 ** -149], dtype=torch.float32)) != 0.0
    g = torch.Generator().manual_seed(0)
    n = 20000
    a, b, c = _f32_values(g, n), _f32_values(g, n), _f32_values(g, n)
    # products near the subnormal range and sums of nearly cancelling terms
    b[n // 2:] = _f32_values(g, n - n // 2).abs().clamp(2.0 ** -30, 2.0 ** -20)
    c[n // 4: n // 2] = -(a[n // 4: n // 2].double() * b[n // 4: n // 2].double()).float()
    an, bn, cn = a.numpy(), b.numpy(), c.numpy()
    with np.errstate(all="ignore"):
        for f, ref in ((add, an + bn), (mul, an * bn), (div, an / bn)):
            assert np.array_equal(bits(f(a, b)).numpy(), ref.view(np.int32)), f.__name__
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.fmaf.restype, libm.fmaf.argtypes = ctypes.c_float, [ctypes.c_float] * 3
    ref = np.array([libm.fmaf(float(x), float(y), float(z)) for x, y, z in zip(an, bn, cn)], dtype=np.float32)
    got = fmaf32(a, b, c).numpy()
    assert np.array_equal(got.view(np.int32), ref.view(np.int32))
    sub = np.abs(ref) < 2.0 ** -126
    print("\nrounding helpers: %d fmaf, add, mul and div checks each, %d fmaf results subnormal" % (n, int((sub & (ref != 0)).sum())))
    assert int((sub & (ref != 0)).sum()) > 100


def test_oracle_and_reference_goldens_lie_within_the_bound():
    """The reference's goldens (their F.conv2d order) and the oracle's LAFs against the float64 soft-argmax of the same inputs."""
    for name, pyr, sig, seq, ref, ora, maps in DC.golden_rows():
        R = Restated(pyr, sig, seq, None, maps=maps)
        rr, ro = bound_ratio(ref, R.lafs64, R.bound), bound_ratio(ora, R.lafs64, R.bound)
        print("\n%s: %d rows, worst error / bound: reference %.3f, oracle %.3f" % (name, seq.numel(), rr, ro))
        assert rr <= 1.0 and ro <= 1.0, name


def _cases():
    """(name, pyr, sigmas, mr, th) of the cases whose candidates the GPU tests pin: the graf crop, the seam pyramid at borders 0
    and 1, the low-contrast pyramid at every k and in threshold mode."""
    pyr, sig, _ = O.scale_pyramid(gray_from_rgb(gold("graf_crop.npz")["rgb"]))
    out = [("graf crop", pyr, sig, MR, 0.0), ("graf crop th 5", pyr, sig, MR, 5.0)]
    _, ssig, spyr = DC.seam_case()
    out += [("seams border %d" % b, spyr, ssig, float(b), 0.0) for b in (0, 1)]
    _, lsig, lpyr = DC.low_contrast_case()
    out += [("low contrast k %d" % k, DC.scaled(lpyr, k), lsig, MR, 0.0) for k in DC.LOW_K]
    return out


@pytest.fixture(scope="module")
def cases():
    return [(name, OracleCandidates(pyr, sig, mr, th)) for name, pyr, sig, mr, th in _cases()]


def test_both_orders_lie_within_the_bound(cases):
    worst = {o: 0.0 for o in ORDERS}
    differ = total = 0
    for name, c in cases:
        R = {o: Restated(c.pyr, c.sigmas, c.seq, o, th=c.th) for o in ORDERS}
        for o in ORDERS:
            worst[o] = max(worst[o], bound_ratio(R[o].lafs32, R[o].lafs64, R[o].bound))
        worst_o = bound_ratio(c.lafs, R["rows"].lafs64, R["rows"].bound)
        assert worst_o <= 1.0, (name, worst_o)
        differ += int((bits(R["rows"].lafs32) != bits(R["taps"].lafs32)).any(2).any(1).sum())
        total += c.total
    print("\nsoft-argmax orders on %d candidates: worst error / bound rows %.3f, taps %.3f; the orders differ on %d rows"
          % (total, worst["rows"], worst["taps"], differ))
    assert max(worst.values()) <= 1.0 and differ > 100


def test_gpu_cases_reach_the_edges(cases):
    """The seam pyramid puts candidates on the first and last output column of strips and the first and last row of bands, and on
    all four image edges at border 0; the low-contrast pyramids make den fall on both sides of 1e-8, subnormal taps and plateau
    maxima, and at k >= 14 every positive pixel inside the border becomes a candidate."""
    got = {}
    for name, c in cases:
        got[name] = DC.reach(c.pyr, c.sigmas, c.seq, c.th)
        print("\n%s: %d candidates, %s" % (name, c.total, got[name]))
    s0, s1 = got["seams border 0"], got["seams border 1"]
    for k in ("strip_first", "strip_last", "band_first", "band_last", "top", "bottom", "left", "right"):
        assert s0[k] > 0, k
    for k in ("strip_first", "strip_last", "band_first", "band_last"):
        assert s1[k] > 0, k
    low = [got["low contrast k %d" % k] for k in DC.LOW_K]
    assert sum(x["den_below"] for x in low) > 1000 and sum(x["den_above"] for x in low) > 1000
    assert got["low contrast k 66"]["subnormal"] > 1000 and got["low contrast k 60"]["subnormal"] > 0
    assert got["low contrast k 20"]["plateau"] > 1000
    dense = dict(cases)["low contrast k 16"]
    n_inner = sum((h - 2 * 5) * (w - 2 * 5) for (h, w) in [tuple(o[0].shape[-2:]) for o in dense.pyr])
    assert dense.total > 2.5 * n_inner, (dense.total, n_inner)


def test_mutations_change_the_bits_of_the_gpu_cases(cases):
    """Each deliberately wrong restatement must change at least one LAF row's bits on the cases, in either order."""
    caught = {}
    for m in MUTATIONS:
        for o in ORDERS:
            n = 0
            for name, c in cases:
                a = 5.192 if m == "scale_first" else 1.0
                good = Restated(c.pyr, c.sigmas, c.seq, o, a_scale=a, th=c.th).lafs32
                if m == "swap_order":
                    bad = Restated(c.pyr, c.sigmas, c.seq, "taps" if o == "rows" else "rows", a_scale=a, th=c.th).lafs32
                else:
                    bad = Restated(c.pyr, c.sigmas, c.seq, o, a_scale=a, th=c.th, mutate=m).lafs32
                n += int((bits(good) != bits(bad)).any(2).any(1).sum())
            caught[(m, o)] = n
            assert n > 0, (m, o)
    print("\nmutations caught (rows with changed bits): %s" % caught)
