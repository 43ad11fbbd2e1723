"""CPU tests of the keypoint-geometry restatement (tests/geometry_restated.py): it equals the reference's fp32 torch operations bit for
bit, reproduces the reference's own goldens, and the constructed cases (tests/geometry_cases.py) separate it from the arithmetic the
kernels used before they stopped fusing the 2x2 products, so the GPU tests (tests/test_gpu_geometry.py) can fail."""
import numpy as np
import pytest
import torch

import affnet_oracle as O
import geometry_cases as K
import geometry_restated as G
import scale_space_restated as R
from helpers import gold

MR_SIZE = 5.192
SHAPES = ((97, 127), (127, 97), (767, 1023), (1023, 767), (1920, 1080), (1080, 1920), (320, 256))


def same_bits(a, b):
    """Bit-identical fp32 arrays, where any NaN equals any NaN."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(((a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))).all())


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def fused_mat2(A, B):
    """The 2x2 product as geometry.cu wrote it before: fmaf(a0, b0, fl(a1 * b2)) per entry."""
    A, B = G.f32(A), G.f32(B)
    out = np.empty(A.shape, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(2):
            for j in range(2):
                out[:, i, j] = R.fmaf32(A[:, i, 0], B[:, 0, j], A[:, i, 1] * B[:, 1, j])
    return out


def fused_compose(A, L):
    out = G.f32(L).copy()
    out[:, :, :2] = fused_mat2(A, G.f32(L)[:, :, :2])
    return out


def kernel_touch_ok_before(NL):
    c = K.corner_fused_order(NL)
    with np.errstate(invalid="ignore"):
        return ~((c > 1) | (c < 0)).any(axis=(1, 2))


def product_inputs():
    """(A, B, L): random full-mantissa blocks, the constructed shape rows and the eigen cases (inf / NaN included)."""
    n = 20000
    A = K.random_full(4 * n, 1).reshape(n, 2, 2)
    B = K.random_full(4 * n, 2).reshape(n, 2, 2)
    L = K.random_full(6 * n, 3).reshape(n, 2, 3)
    As, Ls, _ = K.shape_rows(600, 4)
    Ae, Le, _ = K.eigen_cases()
    return np.concatenate([A, As, Ae]), np.concatenate([B, As[::-1], Ae[::-1]]), np.concatenate([L, Ls, Le])


# ---- the restatement is the reference's torch arithmetic --------------------------------------------------------------------------
def test_products_equal_torch_bmm():
    A, B, L = product_inputs()
    assert same_bits(G.mat2(A, B), torch.bmm(t(A), t(B)).numpy())
    assert same_bits(G.compose(A, L), torch.cat([torch.bmm(t(A), t(L)[:, :, :2]), t(L)[:, :, 2:]], 2).numpy())
    assert same_bits(G.rotate(L, B), torch.cat([torch.bmm(t(L)[:, :, :2], t(B)), t(L)[:, :, 2:]], 2).numpy())


def abs_delta1(A):
    A = G.f32(A)
    with np.errstate(invalid="ignore", over="ignore"):
        tr = A[:, 0, 0] + A[:, 1, 1]
        return np.abs(tr * tr - np.float32(4) * (A[:, 0, 0] * A[:, 1, 1] - A[:, 1, 0] * A[:, 0, 1]))


def test_eigen_and_boundary_equal_the_oracle():
    """batch_eig2x2, the ratio test and checkTouchBoundary as the oracle's torch statements compute them, including NaN positions.

    The one exception is the square root: the restatement's (numpy's, and the kernels' __fsqrt_rn) is correctly rounded, while torch's
    vectorised CPU sqrt is 1 ulp off for a fraction of a percent of the arguments on some builds.  Rows where it is are compared for
    their decisions only, and there must be few of them."""
    A, _, L = product_inputs()
    sets = [(A, L), K.boundary_exact()[:2], K.boundary_association(), K.eigen_cases()[:2], K.shape_rows(4000, 9)[:2]]
    off, flips = 0, 0
    for Ai, Li in sets:
        d = abs_delta1(Ai)
        with np.errstate(invalid="ignore"):
            assert same_bits(np.sqrt(d), np.sqrt(d.astype(np.float64)).astype(np.float32)), "numpy's fp32 sqrt is correctly rounded"
        ieee = torch.sqrt(t(d)).numpy().view(np.int32) == np.sqrt(d).view(np.int32)
        ieee |= np.isnan(d)
        l1, l2 = G.batch_eig2x2(Ai)
        o1, o2 = O.batch_eig2x2(t(Ai))
        assert same_bits(l1[ieee], o1.numpy()[ieee]) and same_bits(l2[ieee], o2.numpy()[ieee])
        NL = G.compose(Ai, Li)
        assert same_bits(G.corners(NL), torch.matmul(t(NL), torch.tensor([[-1., -1, 1, 1], [-1, 1, -1, 1], [1, 1, 1, 1]])).numpy())
        assert np.array_equal(G.touch_ok(NL), O.check_touch_boundary(t(NL)).numpy())
        m, om = G.shape_mask(Ai, Li), O.shape_filter_mask(t(Ai), t(NL)).numpy()
        assert np.array_equal(m[ieee], om[ieee])
        off += int((~ieee).sum()); flips += int((m != om).sum())
    print("\ntorch.sqrt not correctly rounded on %d rows; %d decisions differ there" % (off, flips))
    assert off < 0.01 * len(A) and flips <= 2


def test_constructed_decisions():
    """The boundary rows decide as constructed (0 and 1 inclusive), and each eigen case lands where it is named."""
    A, L, keep = K.boundary_exact()
    assert np.array_equal(G.shape_mask(A, L), keep)
    found = K.ratio_neighbours()
    for r, a in found.items():
        assert float(G.eig_ratio(a[None])[0]) == r and bool(G.eig_ok(a[None])[0]) == (G.SIXTH < r < 6)
    assert set(found) == {float(K.ulps(v, k)) for v in (np.float32(6), G.SIXTH) for k in (-1, 0, 1)}
    A, L, names = K.eigen_cases()
    ratio, ok = G.eig_ratio(A), G.shape_mask(A, L)
    by = dict(zip(names, zip(ratio, ok)))
    assert np.isinf(by["l2 = -1e-8 (ratio inf)"][0]) and not by["l2 = -1e-8 (ratio inf)"][1]
    assert by["det < 0, l = 1, -2"][1] and by["both negative, ratio 1/3"][1] and not by["det < 0, l = -6, 1"][1]
    assert not any(by[n][1] for n in names if n.startswith(("identity", "2I", "rotation", "similarity", "det = 0", "A ")))
    assert by["LAF NaN centre"][1] and by["LAF NaN shape"][1], "NaN corners pass checkTouchBoundary in the reference"
    assert not by["LAF inf centre"][1] and not by["LAF -inf shape"][1]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_selection_equals_torch_topk(seed):
    """select() returns torch.topk's values of resp * mask when survivors exceed num_features (the rows wherever the value is unique),
    and the survivors in row order otherwise."""
    A, L, resp = K.shape_rows(3000, 100 + seed)
    mask = G.shape_mask(A, L)
    S = int(mask.sum())
    for nf in (0, 1, 7, S // 2, S - 1, S, S + 1):
        rows, vals = G.select(mask, resp, nf, len(resp))
        if nf > 0 and S > nf:
            key = t(resp) * t(mask).float()
            v, _ = torch.topk(key, nf)
            assert torch.equal(t(vals), v)
            u, c = np.unique(key.numpy(), return_counts=True)
            uniq = np.isin(vals, u[c == 1])
            assert np.array_equal(rows[uniq], np.array([int(np.nonzero(key.numpy() == x)[0][0]) for x in vals[uniq]], dtype=rows.dtype))
        else:
            assert np.array_equal(rows, np.nonzero(mask)[0]) and same_bits(vals, resp[mask])
    # ties: equal values come out lowest row first
    rows, vals = G.select(mask, resp, S // 2, len(resp))
    for a, b, ra, rb in zip(vals[:-1], vals[1:], rows[:-1], rows[1:]):
        assert a > b or (a == b and ra < rb)


def test_response_case_reaches_the_zeros():
    """The response case is sharp: its cuts put rejected rows (as zeros) ahead of negative survivors, a -0.0 survivor ties the zeros, and
    writing the raw response of a selected rejected row would differ from the reference's value."""
    A, L, resp, keep = K.response_case()
    assert np.array_equal(G.shape_mask(A, L), keep)
    hit = 0
    for nf in K.RESPONSE_NF:
        rows, vals = G.select(keep, resp, nf, len(resp))
        v, _ = torch.topk(t(resp) * t(keep).float(), nf) if keep.sum() > nf else (t(resp[keep]), None)
        assert torch.equal(t(vals), v)
        hit += int((~keep[rows] & (resp[rows] != 0)).any())
    assert hit >= 3


def test_scale_equals_the_oracle():
    L = np.concatenate([K.random_lafs(5000, 7), K.eigen_cases()[1]])
    for (w, h) in SHAPES:
        assert same_bits(G.scale(L, *G.denorm_coefs(w, h)), O.denormalize_lafs(t(L), w, h).numpy())
        assert same_bits(G.scale(L, *G.norm_coefs(w, h)), O.normalize_lafs(t(L), w, h).numpy())
        # the pipeline's coefficients (pipeline.cu): 1.0f / ms, (float)(1.0 / W), (float)(1.0 / H)
        ms = np.float32(min(w, h))
        assert G.norm_coefs(w, h) == (np.float32(1.0) / ms, np.float32(1.0 / w), np.float32(1.0 / h))


# ---- the reference's goldens --------------------------------------------------------------------------------------------------------
def golden_shape_inputs():
    z = gold("graf_crop.npz")
    L = z["det_LAFs"].copy()
    L[:, :, :2] = np.float32(MR_SIZE) * L[:, :, :2]           # SparseImgRepresenter.py:198, an fp32 product
    return z, z["aff_A"], z["det_resp"], L, int(z["K"])


def test_goldens_bit_for_bit():
    """shape_LAFs / shape_resp from aff_A and the detector LAFs, and ori_dLAFs = denormalise(rotate(shape_LAFs, ori_R)) at 320x256."""
    z, A, resp, L, Kf = golden_shape_inputs()
    rows, vals, lafs = G.shape_filter(A, resp, L, Kf)
    assert same_bits(vals, z["shape_resp"]) and same_bits(lafs, z["shape_LAFs"])
    assert np.array_equal(z["det_pidx"][rows], z["shape_pidx"]) and np.array_equal(z["det_lidx"][rows], z["shape_lidx"])
    d = G.scale(G.rotate(z["shape_LAFs"], z["ori_R"]), *G.denorm_coefs(320, 256))
    assert same_bits(d, z["ori_dLAFs"])


# ---- the cases can fail the kernels' previous arithmetic -------------------------------------------------------------------------
def test_cases_separate_the_fused_arithmetic():
    z, A, resp, L, Kf = golden_shape_inputs()
    # the orientation golden: the fused rotation misses rows of ori_dLAFs
    fused_rot = G.f32(z["shape_LAFs"]).copy()
    fused_rot[:, :, :2] = fused_mat2(fused_rot[:, :, :2], z["ori_R"])
    fused_d = G.scale(fused_rot, *G.denorm_coefs(320, 256))
    miss = int((~np.all(fused_d.view(np.int32) == z["ori_dLAFs"].view(np.int32), axis=(1, 2))).sum())
    print("\nfused rotation: %d of %d ori_dLAFs rows differ" % (miss, len(fused_d)))
    assert miss >= 50
    # random products: about a quarter of the entries differ
    A2, B2, L2 = product_inputs()
    frac = float((fused_mat2(A2, B2).view(np.int32) != G.mat2(A2, B2).view(np.int32)).mean())
    print("fused 2x2 product: %.3f of the entries differ" % frac)
    assert frac > 0.15
    assert not same_bits(fused_compose(A2, L2), G.compose(A2, L2))
    # the association rows: every one flips its keep decision under h0*x + (h1*y + h2)
    Aa, La = K.boundary_association()
    NL = G.compose(Aa, La)
    assert np.array_equal(NL, fused_compose(Aa, La)), "A_EXACT composes exactly in both forms"
    assert np.all(G.touch_ok(NL) != kernel_touch_ok_before(NL))
    # the shape rows the GPU test uses at cap >= 1024 carry some of them
    As, Ls, _ = K.shape_rows(1024, 1)
    assert (G.shape_mask(As, Ls) != (G.eig_ok(As) & kernel_touch_ok_before(fused_compose(As, Ls)))).sum() >= 100
