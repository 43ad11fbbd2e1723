"""GPU tests (-m gpu): the keypoint-geometry entry points bit for bit against the fp32 restatement of the reference's arithmetic
(tests/geometry_restated.py) on the constructed cases of tests/geometry_cases.py, and LAFs2ellT within a bound derived from its fp32
chain.  Outputs start poisoned or as a sentinel, so a missing or stray write is seen.  tests/test_geometry_cpu.py shows on the CPU that
these cases separate the restatement from fused 2x2 products and from the other association of the corner sums."""
import numpy as np
import pytest
import torch

import affnet_oracle as O
import geometry_cases as K
import geometry_restated as G
from helpers import POISON_INF, SENTINEL, gold, poisoned

pytestmark = pytest.mark.gpu

DEV = "cuda"
AG_ERR_INVALID, AG_ERR_CAPACITY = -1, -3
POISON_WORD = (POISON_INF << 16) | POISON_INF          # every 32-bit output word of a poisoned buffer (fp32 ~2.7e36, not -1)
MAX_CAP = 16384
CAPS = (1, 31, 33, 1024, 1025, 4097, MAX_CAP)          # growing: the shared-memory attribute is raised within one process
SHAPES = ((97, 127), (127, 97), (767, 1023), (1023, 767), (1920, 1080), (1080, 1920))
NS = (1, 255, 256, 257, 65537)
U32 = 2.0 ** -24


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


def same_bits(a, b):
    """Bit-identical fp32 (any NaN equals any NaN: the device's NaN payload is canonical)."""
    a = np.ascontiguousarray(a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a, np.float32)
    b = np.ascontiguousarray(b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else b, np.float32)
    return a.shape == b.shape and bool(((a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))).all())


def dev(x, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV, dtype).contiguous()


def poisoned_out(shape, dtype):
    n = int(np.prod(shape))
    return poisoned(4 * n, POISON_INF).view(dtype).view(*shape)


def untouched(x):
    """Every 32-bit word of x still holds the poison."""
    return bool((x.contiguous().view(torch.int32) == POISON_WORD).all())


def shape_filter(L, A, Lf, resp, octs, lvls, counts, cap, nf, out_cap, B=None):
    """ag_affine_shape_filter on [B,cap] inputs into poisoned outputs -> (rc, resp, lafs, oct, lvl, count)."""
    B = len(counts) if B is None else B
    nb, nr = max(B, 1), max(out_cap, 1)
    outs = (poisoned_out((nb, nr), torch.float32), poisoned_out((nb, nr, 2, 3), torch.float32), poisoned_out((nb, nr), torch.int32),
            poisoned_out((nb, nr), torch.int32), poisoned_out((nb,), torch.int32))
    ci = torch.tensor(list(counts) or [0], dtype=torch.int32, device=DEV)
    rc = L.lib().ag_affine_shape_filter(L.ptr(A), L.ptr(resp), L.ptr(Lf), L.ptr(octs), L.ptr(lvls), L.ptr(ci), B, cap, nf, out_cap,
                                        *[L.ptr(o) for o in outs], L.stream_ptr())
    torch.cuda.synchronize()
    return (rc,) + outs


def batch_inputs(cap, counts, seed):
    """B images of `cap` rows: every image starts with the constructed rows, then random ones (a different draw per image)."""
    rows = [K.shape_rows(cap, seed + 13 * b) for b in range(len(counts))]
    A = np.stack([r[0] for r in rows]); Lf = np.stack([r[1] for r in rows]); resp = np.stack([r[2] for r in rows])
    octs = np.arange(len(counts) * cap, dtype=np.int32).reshape(len(counts), cap) % 7
    lvls = (np.arange(len(counts) * cap, dtype=np.int32).reshape(len(counts), cap) * 3 + 1) % 5
    return A, Lf, resp, octs, lvls


def check_filter(out, A, Lf, resp, octs, lvls, counts, cap, nf, out_cap):
    """Every image's outputs against the restatement; rows at or beyond the count stay poisoned.  -> survivors per image."""
    rc, ro, lo, oo, vo, co = out
    assert rc == 0
    S = []
    for b, c in enumerate(counts):
        n = max(0, min(c, cap))
        rows, vals, lafs = G.shape_filter(A[b, :n], resp[b, :n], Lf[b, :n], nf, out_cap)
        m = len(rows)
        S.append(int(G.shape_mask(A[b, :n], Lf[b, :n]).sum()))
        tag = (cap, nf, out_cap, b, c)
        assert int(co[b]) == (-1 if c < 0 else m), tag
        assert same_bits(ro[b, :m], vals), tag
        assert same_bits(lo[b, :m], lafs), (tag, int((lo[b, :m].cpu().numpy() != lafs).any(axis=(1, 2)).sum()))
        assert np.array_equal(oo[b, :m].cpu().numpy(), octs[b, rows]) and np.array_equal(vo[b, :m].cpu().numpy(), lvls[b, rows]), tag
        assert untouched(ro[b, m:]) and untouched(lo[b, m:]) and untouched(oo[b, m:]) and untouched(vo[b, m:]), tag
    return S


# ---- ag_affine_shape_filter ---------------------------------------------------------------------------------------------------------
def test_shape_filter_batched_every_cap(L):
    """B = 5 ragged images (full, 0, -1, above cap, two thirds) at every cap in growing order; num_features 0, S - 1, S, S + 1 of the first
    image and out_cap at cap and below the survivors; then B = 1..4 at cap 1025."""
    for cap in CAPS:
        counts = [cap, 0, -1, cap + 5, max(1, 2 * cap // 3)]
        A, Lf, resp, octs, lvls = batch_inputs(cap, counts, cap)
        d = (dev(A), dev(Lf), dev(resp), dev(octs, torch.int32), dev(lvls, torch.int32))
        S0 = int(G.shape_mask(A[0], Lf[0]).sum())
        for nf in sorted({0, S0 - 1, S0, S0 + 1}):
            for out_cap in sorted({cap, max(1, S0 // 2)}):
                out = shape_filter(L, *d, counts, cap, nf, out_cap)
                check_filter(out, A, Lf, resp, octs, lvls, counts, cap, nf, out_cap)
        print("\ncap %5d: %d survivors of %d rows in image 0" % (cap, S0, cap))
    cap = 1025
    for B in (1, 2, 3, 4):
        counts = [cap, 700, -1, 0][:B]
        A, Lf, resp, octs, lvls = batch_inputs(cap, counts, 77 + B)
        d = (dev(A), dev(Lf), dev(resp), dev(octs, torch.int32), dev(lvls, torch.int32))
        for nf in (0, 100):
            check_filter(shape_filter(L, *d, counts, cap, nf, cap), A, Lf, resp, octs, lvls, counts, cap, nf, cap)


def test_shape_filter_response_ties_and_zeros(L):
    """Tied responses at the cut, -0.0, and rejected rows that enter the top K as zeros ahead of negative survivors."""
    A, Lf, resp, keep = K.response_case()
    n = len(keep)
    octs, lvls = np.arange(n, dtype=np.int32)[None], (np.arange(n, dtype=np.int32)[None] * 5) % 3
    d = (dev(A), dev(Lf), dev(resp), dev(octs, torch.int32), dev(lvls, torch.int32))
    for nf in K.RESPONSE_NF:
        for out_cap in (n, 3):
            check_filter(shape_filter(L, *d, [n], n, nf, out_cap), A[None], Lf[None], resp[None], octs, lvls, [n], n, nf, out_cap)


def test_shape_filter_refusals(L):
    """cap 16385 needs more shared memory than the sort has: AG_ERR_CAPACITY, nothing written.  B, cap or out_cap of 0: AG_ERR_INVALID."""
    cap = MAX_CAP + 1
    A, Lf, resp, octs, lvls = batch_inputs(cap, [cap], 3)
    d = (dev(A), dev(Lf), dev(resp), dev(octs, torch.int32), dev(lvls, torch.int32))
    rc, *outs = shape_filter(L, *d, [cap], cap, 10, cap)
    assert rc == AG_ERR_CAPACITY and all(untouched(o) for o in outs)
    for B, c, oc in ((0, 8, 8), (1, 0, 8), (1, 8, 0)):
        rc, *outs = shape_filter(L, *d, [8], c, 4, oc, B=B)
        assert rc == AG_ERR_INVALID and all(untouched(o) for o in outs), (B, c, oc)


# ---- the other entry points ---------------------------------------------------------------------------------------------------------
def product_inputs(n, seed):
    """n rows of full-mantissa blocks with the eigen cases (inf / NaN entries) and the goldens' R spliced in."""
    A = K.random_full(4 * n, seed).reshape(n, 2, 2)
    B = K.random_full(4 * n, seed + 1).reshape(n, 2, 2)
    Lf = K.random_full(6 * n, seed + 2).reshape(n, 2, 3)
    Ae, Le, _ = K.eigen_cases()
    k = min(n, len(Ae))
    A[n - k:], Lf[n - k:] = Ae[:k], Le[:k]
    B[:min(n, 300)] = gold("graf_crop.npz")["ori_R"][:min(n, 300)]
    return A, B, Lf


def padded(x, pad=5):
    """x on the device followed by `pad` rows of SENTINEL."""
    out = torch.full((x.shape[0] + pad,) + x.shape[1:], SENTINEL, device=DEV)
    out[:x.shape[0]] = dev(x)
    return out


@pytest.mark.parametrize("n", NS)
def test_products_and_scale_bit_exact(L, n):
    lib = L.lib()
    A, B, Lf = product_inputs(n, n)
    dA, dB, dL = dev(A), dev(B), dev(Lf)
    # ag_lafs_apply_rotation, in place: rows past n keep the sentinel
    x = padded(Lf); x[n:] = SENTINEL
    L.check(lib.ag_lafs_apply_rotation(L.ptr(x), L.ptr(dB), n, L.stream_ptr()))
    torch.cuda.synchronize()
    assert same_bits(x[:n], G.rotate(Lf, B)) and bool((x[n:] == SENTINEL).all())
    # ag_mat2_compose and ag_lafs_left_multiply
    o = padded(np.zeros((n, 2, 2), np.float32)); o[:] = SENTINEL
    L.check(lib.ag_mat2_compose(L.ptr(dA), L.ptr(dB), L.ptr(o), n, L.stream_ptr()))
    torch.cuda.synchronize()
    assert same_bits(o[:n], G.mat2(A, B)) and bool((o[n:] == SENTINEL).all())
    o = padded(np.zeros((n, 2, 3), np.float32)); o[:] = SENTINEL
    L.check(lib.ag_lafs_left_multiply(L.ptr(dA), L.ptr(dL), L.ptr(o), n, L.stream_ptr()))
    torch.cuda.synchronize()
    assert same_bits(o[:n], G.left_multiply(A, Lf)) and bool((o[n:] == SENTINEL).all())
    # ag_lafs_scale with both coefficient sets
    for (w, h) in SHAPES[::2]:
        for coefs in (G.denorm_coefs(w, h), G.norm_coefs(w, h)):
            o[:] = SENTINEL
            L.check(lib.ag_lafs_scale(L.ptr(dL), L.ptr(o), n, *[float(c) for c in coefs], L.stream_ptr()))
            torch.cuda.synchronize()
            assert same_bits(o[:n], G.scale(Lf, *coefs)) and bool((o[n:] == SENTINEL).all()), (w, h)


def test_normalize_denormalize_through_laf(L):
    """LAF.normalizeLAFs / denormalizeLAFs at landscape and portrait sizes against the reference's coefficient products."""
    from affnet_b200.LAF import denormalizeLAFs, normalizeLAFs
    Lf = np.concatenate([K.random_lafs(4097, 5), K.eigen_cases()[1]])
    for (w, h) in SHAPES:
        assert same_bits(denormalizeLAFs(dev(Lf), w, h), G.scale(Lf, *G.denorm_coefs(w, h))), (w, h)
        assert same_bits(normalizeLAFs(dev(Lf), w, h), G.scale(Lf, *G.norm_coefs(w, h))), (w, h)
        assert same_bits(normalizeLAFs(dev(Lf), w, h), O.normalize_lafs(torch.from_numpy(Lf), w, h)), (w, h)


def test_zero_rows_write_nothing(L):
    lib = L.lib()
    x = torch.full((4, 2, 3), SENTINEL, device=DEV); r = torch.zeros(4, 2, 2, device=DEV)
    for rc in (lib.ag_lafs_apply_rotation(L.ptr(x), L.ptr(r), 0, L.stream_ptr()), lib.ag_mat2_compose(L.ptr(r), L.ptr(r), L.ptr(x), 0, L.stream_ptr()),
               lib.ag_lafs_left_multiply(L.ptr(r), L.ptr(x), L.ptr(x), 0, L.stream_ptr()),
               lib.ag_lafs_scale(L.ptr(r), L.ptr(x), 0, 1.0, 1.0, 1.0, L.stream_ptr())):
        assert rc == 0
    torch.cuda.synchronize()
    assert bool((x == SENTINEL).all())


# ---- the reference's own chain ------------------------------------------------------------------------------------------------------
def test_reference_chain_bit_for_bit(L):
    """With the reference's A: shape filter -> rotation by ori_R -> denormalise gives the reference's shape_LAFs, shape_resp and
    ori_dLAFs bit for bit (the rotation known answer: fused products miss a third of its rows)."""
    lib = L.lib()
    z = gold("graf_crop.npz")
    Kf = int(z["K"])
    Lf = z["det_LAFs"].copy(); Lf[:, :, :2] = np.float32(5.192) * Lf[:, :, :2]
    n = len(Lf)
    octs, lvls = z["det_pidx"].astype(np.int32)[None], z["det_lidx"].astype(np.int32)[None]
    d = (dev(z["aff_A"]), dev(Lf), dev(z["det_resp"]), dev(octs, torch.int32), dev(lvls, torch.int32))
    rc, ro, lo, oo, vo, co = shape_filter(L, *d, [n], n, Kf, Kf)
    assert rc == 0 and int(co[0]) == Kf
    assert same_bits(ro[0], z["shape_resp"]) and same_bits(lo[0], z["shape_LAFs"])
    assert np.array_equal(oo[0].cpu().numpy(), z["shape_pidx"]) and np.array_equal(vo[0].cpu().numpy(), z["shape_lidx"])
    lafs = lo[0].clone()
    L.check(lib.ag_lafs_apply_rotation(L.ptr(lafs), L.ptr(dev(z["ori_R"])), Kf, L.stream_ptr()))
    out = torch.empty_like(lafs)
    L.check(lib.ag_lafs_scale(L.ptr(lafs), L.ptr(out), Kf, *[float(c) for c in G.denorm_coefs(320, 256)], L.stream_ptr()))
    torch.cuda.synchronize()
    assert same_bits(out, z["ori_dLAFs"]), int((out.cpu().numpy() != z["ori_dLAFs"]).any(axis=(1, 2)).sum())


# ---- ag_lafs_to_ell ---------------------------------------------------------------------------------------------------------------------
ELL_C = 32.0   # error of the ellipse matrix relative to its largest entry <= ELL_C * u * (1 + elongation^2): see DESIGN.md


def test_lafs_to_ell_vs_float64(L):
    """LAFs2ellT on the device against the reference's closed form in float64.  The small singular value comes from
    sqrt((sum - dif) / 2), whose fp32 cancellation costs a relative u * elongation^2; the bound is ELL_C times that.  NaN and inf
    appear where the fp32 torch statement (the oracle) has them."""
    from affnet_b200.LAF import LAFs2ellT
    Ls, elong = K.ell_cases()
    e = LAFs2ellT(dev(Ls)).cpu().numpy()
    r32 = O.lafs_to_ell_t(torch.from_numpy(Ls)).numpy()
    assert np.array_equal(np.isnan(e), np.isnan(r32)) and np.array_equal(np.isinf(e), np.isinf(r32))
    assert np.array_equal(e[:, 0], Ls[:, 0, 2]) and np.array_equal(e[:, 1], Ls[:, 1, 2])
    ok = np.isfinite(r32).all(axis=1)
    assert ok.sum() >= len(Ls) - 4 and (~ok).sum() == 4     # the three LAFs with det < 0 and the zero LAF
    r64 = G.lafs_to_ell64(Ls)[ok]
    err = np.abs(e[ok, 2:] - r64[:, 2:]).max(axis=1) / np.abs(r64[:, 2:]).max(axis=1)
    bound = ELL_C * U32 * (1 + elong[ok] ** 2)
    w = int(np.argmax(err / bound))
    print("\nLAFs2ellT: worst error %.2e at elongation %.4g (%.2f of its bound); worst at elongation < 6: %.2e" % (
        err[w], elong[ok][w], err[w] / bound[w], err[elong[ok] < 6].max()))
    assert np.all(err <= bound)
