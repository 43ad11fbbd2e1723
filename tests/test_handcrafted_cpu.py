"""CPU tests: the fp32 restatement of the hand-crafted estimators and the SIFT descriptor (tests/handcrafted_restated.py), run with
correctly rounded atan2, against the unmodified reference's outputs (tests/golden/handcrafted.npz, sift.npz, handcrafted_edges.npz),
and mutation checks showing that the bit-exact GPU tests built on it see a wrong operation order or a fused multiply-add."""
import numpy as np
import pytest
import torch

import handcrafted_restated as H
import oracle_sift as OS
from helpers import gold, orientation_boundary_shares

U = 2.0 ** -24
HC_PS = (3, 5, 15, 19, 32, 41)
SIFT_PS = (16, 32, 41, 65)


@pytest.fixture(scope="module")
def edges():
    return gold("handcrafted_edges.npz")


def nan_equal(a, b):
    return np.array_equal(np.isnan(a), np.isnan(b))


def baumberg64(P, gk):
    """AffineShapeEstimator in float64 (gradients are exact there) -> (A [n,2,2], the moments (a, b, c) and the sums of their terms'
    magnitudes, both / NP)."""
    P = np.asarray(P, np.float64)
    n, PS = P.shape[0], P.shape[-1]
    idx = np.arange(PS)
    m, p = np.maximum(idx - 1, 0), np.minimum(idx + 1, PS - 1)
    gx, gy = P[:, :, p] - P[:, :, m], P[:, p, :] - P[:, m, :]
    g = np.asarray(gk, np.float64)
    with np.errstate(all="ignore"):
        t = [(u * v * g).reshape(n, -1) for u, v in ((gx, gx), (gx, gy), (gy, gy))]
        return [x.mean(axis=1) for x in t], [np.abs(x).mean(axis=1) for x in t]


def inv_sqrt_rectify64(a, b, c):
    with np.errstate(all="ignore"):
        mask = (b != 0).astype(np.float64)
        r1 = mask * (c - a) / (2.0 * b + 1e-12)
        t1 = np.sign(r1) / (np.abs(r1) + np.sqrt(1.0 + r1 * r1))
        r = 1.0 / np.sqrt(1.0 + t1 * t1)
        t = t1 * r
        r = r * mask + (1.0 - mask)
        t = t * mask
        x = 1.0 / np.sqrt(r * r * a - 2.0 * r * t * b + t * t * c)
        z = 1.0 / np.sqrt(t * t * a + 2.0 * r * t * b + r * r * c)
        d = np.sqrt(x * z)
        x, z = x / d, z / d
        na, nb, nc = r * r * x + t * t * z, -r * t * x + t * r * z, t * t * x + r * r * z
        det = np.sqrt(np.abs(na * nc - nb * nb + 1e-10))
        b2a2 = np.sqrt(nb * nb + na * na)
        return np.stack([b2a2 / det, 0.0 * det, (nc * nb + nb * na) / (b2a2 * det), det / b2a2], axis=1).reshape(-1, 2, 2)


def baumberg_bound(P, gk):
    """(A64, bound [n]): |fp32 Baumberg - A64| <= bound for any fp32 evaluation of the reference's chain.

    Each moment term fl(fl(u v) g) carries at most 4 roundings (the gradient, two products, with fl(gx gy) of two rounded gradients);
    the sum of NP terms by any order of depth <= NP adds gamma_NP of the sum of magnitudes (Higham 4.3), and / NP one rounding.  So
    |a32 - a| <= (NP + 6) u sum|t_a| / NP, and the same for b and c.  That box is propagated through the float64 inverse square root
    by evaluating it at the 8 corners (x 2 against the curvature between them); the fp32 evaluation of that chain adds at most
    64 u max|A| (about 40 roundings, none of them cancelling after the square roots)."""
    PS = P.shape[-1]
    (a, b, c), (sa, sb, sc) = baumberg64(P, gk)
    A64 = inv_sqrt_rectify64(a, b, c)
    k = (PS * PS + 6) * U
    worst = np.zeros(len(a))
    with np.errstate(all="ignore"):
        for ia in (-1, 1):
            for ib in (-1, 1):
                for ic in (-1, 1):
                    Ac = inv_sqrt_rectify64(a + ia * k * sa, b + ib * k * sb, c + ic * k * sc)
                    worst = np.fmax(worst, np.abs(Ac - A64).reshape(len(a), -1).max(axis=1))
        return A64, 2.0 * worst + 64.0 * U * np.abs(A64).reshape(len(a), -1).max(axis=1)


def check_baumberg(P, gk, ref, tag):
    """Restatement and the reference's fp32 output both within baumberg_bound of float64; NaN positions identical."""
    A = H.baumberg(P, gk)
    assert nan_equal(A, ref), (tag, np.argwhere(np.isnan(A) != np.isnan(ref))[:5])
    A64, bd = baumberg_bound(P, gk)
    ok = np.isfinite(A64).all(axis=(1, 2)) & np.isfinite(A).all(axis=(1, 2))
    worst = 0.0
    for X in (A, ref):
        e = np.abs(X[ok] - A64[ok]).reshape(ok.sum(), -1).max(axis=1)
        assert (e <= bd[ok]).all(), (tag, e.max(), bd[ok][np.argmax(e - bd[ok])])
        worst = max(worst, float((e / np.maximum(bd[ok], 1e-30)).max(initial=0.0)))
    return A, float(np.abs(A[ok] - A64[ok]).max(initial=0.0)), worst


def check_angles(P, gk, ref, tag):
    """Identical angles, except where a near-tie or a pixel on a bin boundary decides (helpers.orientation_boundary_shares)."""
    ang = H.orientation_angle(P, gk)
    assert nan_equal(ang, ref), tag
    diff = np.nonzero(ang != ref)[0]
    if len(diff):
        fin = np.isfinite(P[diff]).all(axis=(1, 2))
        assert fin.all(), (tag, diff[~fin])                  # a non-finite patch gives bin 0 on both sides
        margin, share = orientation_boundary_shares(torch.from_numpy(P[diff]).unsqueeze(1))
        assert bool(((share > margin) | (margin == 0)).all()), (tag, diff, margin, share)
    return len(diff)


def test_restated_orientation_matches_reference_graf19():
    z, e = gold("handcrafted.npz"), gold("handcrafted_edges.npz")
    P = z["patches19"][:, 0]
    assert check_angles(P, e["ori_gk_19"], z["angle"], "graf19") == 0


def test_restated_baumberg_matches_reference_graf19():
    z, e = gold("handcrafted.npz"), gold("handcrafted_edges.npz")
    _, err, ratio = check_baumberg(z["patches19"][:, 0], e["aff_gk_19"], z["A"], "graf19")
    print("\nBaumberg graf PS 19: restatement vs float64 %.3g, worst share of the bound %.3f" % (err, ratio))


@pytest.mark.parametrize("PS", HC_PS)
def test_restated_estimators_match_reference_edges(edges, PS):
    P = edges["hc_patches_%d" % PS]
    check_angles(P, edges["ori_gk_%d" % PS], edges["ori_angle_%d" % PS], PS)
    A, err, ratio = check_baumberg(P, edges["aff_gk_%d" % PS], edges["aff_A_%d" % PS], PS)
    print("\nBaumberg PS %d: restatement vs float64 %.3g, worst share of the bound %.3f" % (PS, err, ratio))
    names = list(edges["edge_names"])
    ang = H.orientation_angle(P, edges["ori_gk_%d" % PS])
    # the degenerate semantics the kernels share with the reference
    for nm in ("zero", "constant", "x_ramp", "y_ramp", "nan_pixel", "inf_pixel", "neg_zero"):
        assert np.isnan(A[names.index(nm)]).all(), (PS, nm)
    for nm in ("nan_pixel", "inf_pixel", "neg_inf_pixel"):
        assert ang[names.index(nm)] == np.float32(np.pi), (PS, nm)
    assert ang[names.index("constant")] == 0.0      # every gradient 0: atan2(0, 0) = 0, bin 18
    assert np.isfinite(A[len(names):]).all()


def sift_bound(PS):
    """|fp32 SIFT - float64| per output: the k^2-term pooling of non-negative weights adds gamma_{k^2} of the pooled magnitude and the
    weights themselves about 16 u (the angle split included), relative to the first norm; the two normalisations a few u more; the
    second divides by the norm of the clipped vector, at least clipval = 0.2 of the first's, hence the factor 5."""
    k, _ = H.sift_geometry(PS)
    return 5.0 * (k * k + 64) * U


def check_sift(P, ref, PS, tag):
    gk, pk = OS.sift_windows(PS)
    d = H.sift(P, gk.numpy(), pk.numpy())
    assert nan_equal(d, ref), (tag, np.isnan(d).any(axis=1), np.isnan(ref).any(axis=1))
    ok = ~np.isnan(ref)
    e = float(np.abs(d[ok] - ref[ok]).max(initial=0.0))
    assert e <= 2.0 * sift_bound(PS), (tag, e, sift_bound(PS))
    return e


@pytest.mark.parametrize("PS", SIFT_PS)
def test_restated_sift_matches_reference(edges, PS):
    z = gold("sift.npz")
    worst = 0.0
    for name in ("random", "graf", "constructed"):
        P = OS.golden_patches(z, name, PS)[:, 0].numpy()
        worst = max(worst, check_sift(P, z["%s_desc_%d" % (name, PS)], PS, (name, PS)))
    P = edges["sift_patches_%d" % PS]
    worst = max(worst, check_sift(P, edges["sift_desc_%d" % PS], PS, ("edges", PS)))
    names = list(edges["edge_names"])
    for nm in ("nan_pixel", "inf_pixel", "neg_inf_pixel", "huge"):
        assert np.isnan(edges["sift_desc_%d" % PS][names.index(nm)]).all(), nm   # the reference: all 128 NaN
    print("\nSIFT PS %d: restatement vs reference %.3g (bound %.3g)" % (PS, worst, 2.0 * sift_bound(PS)))


# ---- mutation checks: each wrong restatement disagrees with the right one on a stated share of the cases ------------------------------
def random_patches(PS, n, seed):
    return np.floor(np.random.default_rng(seed).random((n, PS, PS)) * 256.0).astype(np.float32)


@pytest.mark.parametrize("PS", HC_PS)
def test_mutation_contracted_baumberg(edges, PS):
    """The earlier plain-C baumberg_warp left nvcc free to fuse a product into the following add or subtract: the moment accumulation,
    1 + r1^2, 1 + t1^2, r * mask + (1 - mask), both quadratic forms, the three entries of the new matrix, the determinant and the norm.
    Modelled with correctly rounded FMAs at those sites, it changes at least one bit of A on over half the random patches."""
    P = random_patches(PS, 64, PS)
    gk = edges["aff_gk_%d" % PS]
    A, Ac = H.baumberg(P, gk), H.baumberg(P, gk, contract=True)
    share = float((A != Ac).any(axis=(1, 2)).mean())
    print("\nPS %d: contracted Baumberg differs on %.2f of the patches" % (PS, share))
    assert share >= 0.5, share


@pytest.mark.parametrize("PS", HC_PS)
def test_mutation_histogram_order(edges, PS):
    """Summing a bin in reverse raster order changes the bits of a smoothed bin on over a third of the random patches (PS >= 15)."""
    gk = edges["ori_gk_%d" % PS]
    P = random_patches(PS, 32, 7 * PS)
    NP = PS * PS
    v, _ = H.orientation_bins(P, gk)
    vr, _ = H.orientation_bins(P, gk, order=range(NP - 1, -1, -1))
    share = float((v != vr).any(axis=1).mean())
    print("\nPS %d: reversed bin order changes the smoothed bins of %.2f of the patches" % (PS, share))
    if PS >= 15:
        assert share >= 1.0 / 3.0, share


@pytest.mark.parametrize("PS", SIFT_PS)
def test_mutation_sift_separate_multiply_add(PS):
    """Pooling with a rounded product and a separate add changes at least one of the 128 outputs of nearly every random patch."""
    P = random_patches(PS, 16, 3 * PS)
    gk, pk = OS.sift_windows(PS)
    d = H.sift(P, gk.numpy(), pk.numpy())
    dm = H.sift(P, gk.numpy(), pk.numpy(), fused=False)
    share = float((d != dm).any(axis=1).mean())
    assert share >= 0.9, share


def test_atan2_cr_special_values():
    """The correctly rounded atan2 the CPU tests use has C99's special values (the GPU tests require the same of the device's)."""
    z, inf = 0.0, np.inf
    y = np.array([z, -z, z, -z, 1, -1, inf, -inf, inf, inf, -inf, -inf, 1, -1, 1, -1, np.nan, 1], np.float32)
    x = np.array([z, z, -z, -z, z, -z, 1, 1, inf, -inf, inf, -inf, inf, inf, -inf, -inf, 1, np.nan], np.float32)
    pf = np.float32(np.pi)
    want = [0.0, -0.0, pf, -pf, pf / 2, -pf / 2, pf / 2, -pf / 2, pf / 4, np.float32(3 * np.pi / 4), -pf / 4,
            -np.float32(3 * np.pi / 4), 0.0, -0.0, pf, -pf, np.nan, np.nan]
    got = H.atan2_cr(y, x)
    w = np.array(want, np.float32)
    assert np.array_equal(got.view(np.int32)[~np.isnan(w)], w.view(np.int32)[~np.isnan(w)]) and np.isnan(got[np.isnan(w)]).all()
