"""CPU tests: the oracle's detector on NaN, +inf and -inf pixels and on images that overflow fp32, against the unmodified reference's
goldens (tests/golden/make_golden_nonfinite.py), under the one documented deviation (DESIGN.md §2): a NaN survivor of the NMS is no
keypoint, so the oracle gives the reference's rows without those with a NaN response.  The cases must reach what they claim (a
finite maximum suppressed by a NaN beside it, an infinite response, NaN from inf - inf, an overflowing soft-argmax denominator, a
level dropped because a NaN suppressed one of its two maxima), and each deliberate mistake of the NaN rules must break a case."""
import numpy as np
import pytest
import torch

import affnet_oracle as O
from detect_restated import Restated, bits, bound_ratio, same_bits
from helpers import OracleCandidates, detector_level_stats, gold

MR = 5.192
Z = gold("nonfinite.npz")
CASES = sorted(k[4:] for k in Z.files if k.startswith("img_"))
NMS_CASES = sorted(k[4:-5] for k in Z.files if k.startswith("nms_") and k.endswith("_none"))
MUTATIONS = ("fmaxf", "clamp_drops_nan", "emit_nan")


def pyramid(name):
    img = torch.from_numpy(Z["img_" + name])
    pyr, sig, _ = O.scale_pyramid(img, 3, 1.6, 5)
    if name == "oct1_nan":
        y, x = (int(v) for v in Z["oct1_nan"])
        pyr[1][1] = pyr[1][1].clone()
        pyr[1][1][0, 0, y, x] = float("nan")
    return pyr, sig


def golden_det(name, K):
    return [torch.from_numpy(Z["det%d_%s_%s" % (K, name, k)]) for k in ("resp", "lafs", "pyr", "lvl")]


def finite_rows(det):
    keep = ~torch.isnan(det[0])
    return [t[keep] for t in det]


def oracle_det(name, K, mutate=None):
    pyr, sig = pyramid(name)
    try:
        return list(O.multi_scale_detector(pyr, sig, K, MR, mutate=mutate))
    except ValueError:              # no level of any octave accepted (the reference raises there too)
        return [torch.zeros(0), torch.zeros(0, 2, 3), torch.zeros(0), torch.zeros(0)]


def nms_case(name, mutate=None):
    t = lambda k: torch.from_numpy(Z["nms_%s_%s" % (name, k)]).float().view(1, 1, *Z["nms_%s_cur" % name].shape)  # noqa: E731
    return O.nms3d_and_compose(t("low"), t("cur"), t("high"), 0, Z["nms_%s_omap" % name].copy(), list(Z["nms_scales"]), MR, mutate)


def assert_nms_matches(name, mutate=None):
    r, A, om, idx = nms_case(name, mutate)
    if int(Z["nms_%s_none" % name]):
        assert r is None, name
        return
    assert r is not None, name
    keep = ~np.isnan(Z["nms_%s_resp" % name])
    assert same_bits(r, torch.from_numpy(Z["nms_%s_resp" % name][keep])), name
    assert same_bits(A, torch.from_numpy(Z["nms_%s_lafs" % name][keep])), name
    assert np.array_equal(om, Z["nms_%s_omap_out" % name]), name


def assert_det_matches(name, mutate=None):
    for K in (0, int(Z["topk"])):
        got = oracle_det(name, K, mutate)
        if K == 0:
            want = finite_rows(golden_det(name, 0))
            assert got[0].numel() == want[0].numel(), (name, K, got[0].numel(), want[0].numel())
            for i, (g, w) in enumerate(zip(got, want)):
                if i == 1:      # where a soft-argmax sum overflows, the LAF depends on the summation order: compare the rest
                    ok = torch.isfinite(g).all(2).all(1) & torch.isfinite(w).all(2).all(1)
                    assert torch.equal(torch.isfinite(g).all(2).all(1), torch.isfinite(w).all(2).all(1)), (name, K)
                    g, w = g[ok], w[ok]
                assert same_bits(g, w), (name, K)
        else:
            # top-K of the finite keypoints: the keep-all rows' best K (the reference's own top-K rows without NaN come first)
            allr = finite_rows(golden_det(name, 0))[0]
            if allr.numel() <= K:
                assert same_bits(got[0], allr), (name, K)
            else:
                assert torch.equal(got[0], torch.topk(allr, K).values), (name, K)
            pre = finite_rows(golden_det(name, K))
            n = pre[0].numel()
            for i, (g, w) in enumerate(zip(got, pre)):
                if i != 1 or bool(torch.isfinite(w).all()):
                    assert same_bits(g[:n], w), (name, K)


@pytest.mark.parametrize("name", CASES)
def test_hessian_maps_identical_to_the_reference(name):
    img = torch.from_numpy(Z["img_" + name])
    for i, s in enumerate(Z["hess_sigmas"]):
        got, want = O.hessian_response(img, float(s)), torch.from_numpy(Z["hess_%s_%d" % (name, i)])
        assert same_bits(got, want), (name, float(s))


@pytest.mark.parametrize("name", NMS_CASES)
def test_nms_from_response_maps_identical_to_the_reference(name):
    assert_nms_matches(name)


@pytest.mark.parametrize("name", CASES)
def test_detector_identical_to_the_reference_without_nan_rows(name):
    assert_det_matches(name)


def test_cases_reach_what_they_claim():
    h = lambda name, i=0: torch.from_numpy(Z["hess_%s_%d" % (name, i)])  # noqa: E731
    # an infinite pixel: the reference's zero filter taps give NaN next to it (0 * inf), +inf on the diagonals
    for name in ("pinf", "ninf"):
        assert bool(torch.isnan(h(name)).any()) and bool(torch.isinf(h(name)).any()), name
    # the scaled images: the detector's response maps are finite up to 2^58, hold inf at 2^60 and NaN from inf - inf at 2^63;
    # the unblurred image's maps overflow sooner (at sigma 3.2 from 2^57)
    def pyr_maps(k):
        pyr, sig = pyramid("scale_%d" % k)
        assert bool(torch.isfinite(pyr[0][0]).all()), k
        return torch.cat([O.hessian_response(lv, s).flatten() for o in range(len(pyr)) for lv, s in zip(pyr[o], sig[o])])
    for k in (54, 57, 58):
        assert bool(torch.isfinite(pyr_maps(k)).all()), k
    assert bool(torch.isfinite(h("scale_54", 1)).all()) and not bool(torch.isfinite(h("scale_57", 1)).all())
    m60, m63 = pyr_maps(60), pyr_maps(63)
    assert bool(torch.isinf(m60).any()) and not bool(torch.isnan(m60).any())
    assert bool(torch.isinf(m63).any()) and bool(torch.isnan(m63).any())
    assert bool(torch.isnan(h("scale_63")).any())
    # 2^58: every response finite, but some survivors' soft-argmax sums overflow (NaN LAFs with finite responses)
    r, A = golden_det("scale_58", 0)[:2]
    assert bool(torch.isfinite(r).all()) and bool(torch.isnan(A).any())
    assert not bool(torch.isnan(golden_det("scale_57", 0)[1]).any())
    # NaN pixels: the reference emits NaN survivors, first in its top-K
    for name in ("nan_mid", "nan_edge", "nan_corner", "pinf", "ninf", "scale_61"):
        assert bool(torch.isnan(golden_det(name, 0)[0]).any()) and bool(torch.isnan(golden_det(name, int(Z["topk"]))[0][0])), name
    # a finite maximum beside a NaN is suppressed: without the NaN it survives
    lo, cur, hi = (torch.from_numpy(Z["nms_nan_next_to_max_%s" % k]).view(1, 1, 24, 28) for k in ("low", "cur", "high"))
    _, _, _, idx = O.nms3d_and_compose(lo, cur, hi, 0, np.zeros((24, 28), np.uint8), list(Z["nms_scales"]), MR)
    _, _, _, idx_fmax = O.nms3d_and_compose(lo, cur, hi, 0, np.zeros((24, 28), np.uint8), list(Z["nms_scales"]), MR, "fmaxf")
    assert 8 * 28 + 8 not in idx.tolist() and 8 * 28 + 8 in idx_fmax.tolist()
    # an infinite response: a NaN survivor (0 * inf) in the reference
    assert bool(torch.isnan(torch.from_numpy(Z["nms_inf_centre_resp"])).any())
    # NaN survivors where the octave map was nonzero: the map becomes 0 there
    om_in, om_out = Z["nms_nan_on_omap_omap"], Z["nms_nan_on_omap_omap_out"]
    assert om_in[12, 15] == 3 and om_out[12, 15] == 0
    # level drops: two maxima, one suppressed by a NaN; octave 1's second level loses one of its two maxima to the NaN of level 1
    assert int(Z["nms_nan_drops_level_none"]) == 1
    base_pyr, sig, _ = O.scale_pyramid(torch.from_numpy(Z["img_oct1_nan"]), 3, 1.6, 5)
    pyr, _ = pyramid("oct1_nan")
    before, after = detector_level_stats(base_pyr[1], sig[1], MR), detector_level_stats(pyr[1], sig[1], MR)
    assert before[1][:2] == (2, True) and after[1][:2] == (1, False), (before, after)
    assert not bool(((golden_det("oct1_nan", 0)[2] == 1) & (golden_det("oct1_nan", 0)[3] == 1)).any())


@pytest.mark.parametrize("mutate", MUTATIONS)
def test_each_mutation_of_the_nan_rules_breaks_a_case(mutate):
    caught = []
    for name in NMS_CASES:
        if mutate == "clamp_drops_nan":
            continue                 # the response maps are given: no clamp
        try:
            assert_nms_matches(name, mutate)
        except AssertionError:
            caught.append(name)
    for name in CASES:
        try:
            assert_det_matches(name, mutate)
        except AssertionError:
            caught.append(name)
    print("\nmutation %s: caught by %s" % (mutate, caught))
    assert caught, mutate


def test_restatement_bits_and_bound_on_overflowing_sums():
    """The soft-argmax restatement of both kernel orders on the images scaled by 2^57 (finite), 2^58 (den overflows), 2^60 and 2^63 (inf
    and NaN responses, never inside a survivor's window): the float64 bound holds on every row whose sums are finite in any order."""
    worst = 0.0
    for name in ("scale_57", "scale_58", "scale_60", "scale_63"):
        pyr, sig = pyramid(name)
        c = OracleCandidates(pyr, sig, MR)
        for order in ("taps", "rows"):
            R = Restated(pyr, sig, c.seq, order)
            fin = R.finite
            worst = max(worst, bound_ratio(R.lafs32[fin], R.lafs64[fin], R.bound[fin]))
            assert worst <= 1.0, (name, order)
            assert bound_ratio(c.lafs[fin], R.lafs64[fin], R.bound[fin]) <= 1.0, (name, order)
            assert bool(torch.isfinite(R.lafs32[fin]).all())
            # where every sum stays finite in any order, so does the oracle's F.conv2d
            assert bool(torch.isfinite(c.lafs[fin]).all()), (name, order)
        if name == "scale_58":
            assert int((~fin).sum()) > 0
            # NaN positions identical in both orders and in the oracle
            for order in ("taps", "rows"):
                assert torch.equal(torch.isnan(Restated(pyr, sig, c.seq, order).lafs32), torch.isnan(c.lafs)), order
    print("\nscaled images: worst error / bound of both kernel orders on the rows with finite sums %.3f" % worst)
