"""GPU tests (-m gpu): the hand-crafted orientation and Baumberg estimators (ag_orientation_hist, ag_baumberg_shape and the batched
pipeline's fused pyramid kernels) and the SIFT descriptor bit for bit against the fp32 restatement of tests/handcrafted_restated.py, run
with the device's own atan2f / cosf / sinf from ag_debug_libm; the probe itself within the CUDA Programming Guide's ulp bounds.  NaN
outputs are compared by position.  Outputs start as a sentinel, and rows at or past a count must keep it."""
import ctypes as C

import numpy as np
import pytest
import torch

import affnet_oracle as O
import handcrafted_restated as H
from helpers import gold, orientation_boundary_shares

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = -777.25
HC_PS = (3, 4, 5, 15, 19, 31, 32, 33, 41)
SIFT_REFUSED = (17, 18, 23, 28, 38, 48, 58)
ULP_ATAN2, ULP_SINCOS = 3, 2          # CUDA C++ Programming Guide, single-precision mathematical functions (full range)


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


def dev(x, dt=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV, dt)


def probe(L, y, x):
    """ag_debug_libm on fp32 arrays of one shape -> (atan2f(y, x), cosf(x), sinf(x)) as numpy."""
    shp = np.shape(x)
    dy, dx = dev(np.asarray(y, np.float32).ravel()), dev(np.asarray(x, np.float32).ravel())
    n = dx.numel()
    outs = [torch.full((n,), SENT, device=DEV) for _ in range(3)]
    L.check(L.lib().ag_debug_libm(L.ptr(dy), L.ptr(dx), n, *(L.ptr(o) for o in outs), L.stream_ptr()))
    torch.cuda.synchronize()
    return tuple(o.cpu().numpy().reshape(shp) for o in outs)


def same(a, b):
    """Bit-identical, with NaN against NaN whatever its payload."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    m = ~np.isnan(a)
    return np.array_equal(a[m].view(np.int32), b[m].view(np.int32))


def ori_gk(PS):
    return (np.float32(10.0) * O.circular_gauss_kernel(PS).astype(np.float32)).astype(np.float32)


def aff_gk(PS):
    return O.circular_gauss_kernel(PS, sigma=(PS / 2) / 3.0).astype(np.float32)


# ---- the libm probe -------------------------------------------------------------------------------------------------------------------
def ulps(got, ref64):
    """|got - ref| in units of the fp32 spacing at ref (float64)."""
    sp = np.spacing(np.abs(ref64).astype(np.float32)).astype(np.float64)
    return np.abs(got.astype(np.float64) - ref64) / sp


def test_libm_probe_within_documented_ulps(L):
    rng = np.random.default_rng(5)
    n = 1 << 20
    mag = lambda: np.float32(10.0) ** rng.uniform(-40, 38, n).astype(np.float32)   # noqa: E731  every binade, subnormals included
    sgn = lambda: np.where(rng.random(n) < 0.5, -1.0, 1.0).astype(np.float32)     # noqa: E731
    y = np.concatenate([(sgn() * mag()), rng.uniform(-300, 300, n)]).astype(np.float32)
    x = np.concatenate([(sgn() * mag()), rng.uniform(-300, 300, n)]).astype(np.float32)
    at, co, si = probe(L, y, x)
    with np.errstate(all="ignore"):
        ra = np.arctan2(y.astype(np.float64), x.astype(np.float64))
        rc, rs = np.cos(x.astype(np.float64)), np.sin(x.astype(np.float64))
    ea = ulps(at, ra)
    assert ea.max() <= ULP_ATAN2, (ea.max(), y[np.argmax(ea)], x[np.argmax(ea)])
    ec, es = ulps(co, rc), ulps(si, rs)
    assert ec.max() <= ULP_SINCOS and es.max() <= ULP_SINCOS, (ec.max(), es.max())
    print("\nprobe: atan2f %.2f ulp, cosf %.2f ulp, sinf %.2f ulp (max over %d points)" % (ea.max(), ec.max(), es.max(), 2 * n))


def test_libm_probe_special_values(L):
    z, inf, nan, tiny = 0.0, np.inf, np.nan, np.float32(1e-45)
    vals = np.array([z, -z, 1.0, -1.0, inf, -inf, nan, tiny, -tiny, np.float32(1.2e-38)], np.float32)
    y, x = np.meshgrid(vals, vals, indexing="ij")
    at, co, si = probe(L, y, x)
    special = (y == 0) | (x == 0) | ~np.isfinite(y) | ~np.isfinite(x)
    assert same(at[special], H.atan2_cr(y, x)[special])   # C99 F.9.1.4: signed zeros, +-pi, +-pi/2, +-pi/4, +-3pi/4 and NaN
    assert same(at[:2, :2], np.array([[0.0, np.pi], [-0.0, -np.pi]], np.float32))   # atan2f(+-0, +0) = +-0, atan2f(+-0, -0) = +-pi
    xs = x[0]
    assert np.isnan(co[0][np.isinf(xs) | np.isnan(xs)]).all() and np.isnan(si[0][np.isinf(xs) | np.isnan(xs)]).all()
    assert same(si[0][:2], np.array([0.0, -0.0], np.float32)) and (co[0][:2] == 1.0).all()
    assert same(si[0][7:9], xs[7:9])                     # sinf(x) = x for subnormal x


# ---- ag_orientation_hist / ag_baumberg_shape -------------------------------------------------------------------------------------------
def run_hc(L, P, PS, n_rows):
    """Both estimators on the first n_rows of P [m,PS,PS] into outputs of n_rows + 3 rows that start as the sentinel."""
    lib = L.lib()
    d = dev(P[:max(n_rows, 1)].reshape(-1)) if len(P) else torch.zeros(1, device=DEV)
    ang = torch.full((n_rows + 3,), SENT, device=DEV)
    A = torch.full((n_rows + 3, 2, 2), SENT, device=DEV)
    g1, g2 = dev(ori_gk(PS)), dev(aff_gk(PS))
    L.check(lib.ag_orientation_hist(L.ptr(d), n_rows, PS, L.ptr(g1), L.ptr(ang), L.stream_ptr()))
    L.check(lib.ag_baumberg_shape(L.ptr(d), n_rows, PS, L.ptr(g2), L.ptr(A), L.stream_ptr()))
    torch.cuda.synchronize()
    ang, A = ang.cpu().numpy(), A.cpu().numpy()
    assert (ang[n_rows:] == SENT).all() and (A[n_rows:] == SENT).all()
    return ang[:n_rows], A[:n_rows]


def hc_patches(PS, n, seed):
    rnd = np.floor(np.random.default_rng(seed).random((max(n, 0), PS, PS)) * 256.0).astype(np.float32)
    return np.concatenate([H.edge_patches(PS), rnd])[:n] if n > 3 else rnd[:n]


@pytest.mark.parametrize("PS", HC_PS)
def test_estimators_bit_exact(L, PS):
    for n in (0, 1, 2, 3, 257):
        P = hc_patches(PS, n, PS * 1000 + n)
        ang, A = run_hc(L, P, PS, n)
        if n == 0:
            continue
        atan2 = lambda y, x: probe(L, y, x)[0]   # noqa: E731
        assert same(ang, H.orientation_angle(P, ori_gk(PS), atan2)), (PS, n, np.nonzero(ang != H.orientation_angle(P, ori_gk(PS), atan2)))
        ref = H.baumberg(P, aff_gk(PS))
        assert same(A, ref), (PS, n, [i for i in range(n) if not same(A[i], ref[i])][:8])


def test_estimators_bit_exact_graf19(L):
    P = gold("handcrafted.npz")["patches19"][:, 0]
    ang, A = run_hc(L, P, 19, len(P))
    atan2 = lambda y, x: probe(L, y, x)[0]   # noqa: E731
    assert same(ang, H.orientation_angle(P, ori_gk(19), atan2))
    assert same(A, H.baumberg(P, aff_gk(19)))


@pytest.mark.parametrize("PS", (3, 5, 15, 19, 32, 41))
def test_estimators_match_reference_on_edges(L, PS):
    """The reference's own outputs on the degenerate patches: identical angles (but at exact ties or pixels on a bin boundary),
    NaN exactly where the reference has it (a flat patch, a one-axis ramp, a non-finite pixel: all four entries of A)."""
    z = gold("handcrafted_edges.npz")
    P = z["hc_patches_%d" % PS]
    lib = L.lib()
    d = dev(P.reshape(-1))
    n = len(P)
    ang, A = torch.full((n,), SENT, device=DEV), torch.full((n, 2, 2), SENT, device=DEV)
    g1, g2 = dev(z["ori_gk_%d" % PS]), dev(z["aff_gk_%d" % PS])
    L.check(lib.ag_orientation_hist(L.ptr(d), n, PS, L.ptr(g1), L.ptr(ang), L.stream_ptr()))
    L.check(lib.ag_baumberg_shape(L.ptr(d), n, PS, L.ptr(g2), L.ptr(A), L.stream_ptr()))
    ang, A = ang.cpu().numpy(), A.cpu().numpy()
    ref_a, ref_A = z["ori_angle_%d" % PS], z["aff_A_%d" % PS]
    assert np.array_equal(np.isnan(A), np.isnan(ref_A)), [str(x) for x in np.array(z["edge_names"])]
    diff = np.nonzero(ang != ref_a)[0]
    if len(diff):
        assert np.isfinite(P[diff]).all(), diff
        margin, share = orientation_boundary_shares(torch.from_numpy(P[diff]).unsqueeze(1))
        assert bool(((share > margin) | (margin == 0)).all()), (diff, margin, share)
    ok = np.isfinite(ref_A)
    assert np.abs(A[ok] - ref_A[ok]).max(initial=0.0) < 1e-4


# ---- SIFT -------------------------------------------------------------------------------------------------------------------------------
def sift_windows(L, PS):
    k, s = C.c_int(), C.c_int()
    assert L.lib().ag_sift_windows(PS, None, None, C.byref(k), C.byref(s)) == 0
    gk, pk = np.zeros((PS, PS), np.float32), np.zeros((k.value, k.value), np.float32)
    L.check(L.lib().ag_sift_windows(PS, gk.ctypes.data_as(C.c_void_p), pk.ctypes.data_as(C.c_void_p), C.byref(k), C.byref(s)))
    return gk, pk


@pytest.mark.parametrize("PS", [p for p in range(16, 66) if p not in SIFT_REFUSED])
def test_sift_bit_exact(L, PS):
    n = 16
    rnd = np.floor(np.random.default_rng(PS).random((n, PS, PS)) * 256.0).astype(np.float32)
    P = np.concatenate([H.edge_patches(PS), rnd])
    m = len(P)
    out = torch.full((m + 2, 128), SENT, device=DEV)
    dP = dev(P.reshape(-1))
    L.check(L.lib().ag_sift_describe(L.ptr(dP), m, PS, C.c_float(0.2), L.ptr(out), L.stream_ptr()))
    got = out.cpu().numpy()
    assert (got[m:] == SENT).all()
    gk, pk = sift_windows(L, PS)
    ref = H.sift(P, gk, pk, 0.2, lambda y, x: probe(L, y, x)[0])
    bad = [i for i in range(m) if not same(got[i], ref[i])]
    assert not bad, (PS, bad[:8])


@pytest.mark.parametrize("PS", SIFT_REFUSED)
def test_sift_refused_sizes(L, PS):
    out = torch.full((1, 128), SENT, device=DEV)
    P = torch.zeros(PS * PS, device=DEV)
    assert L.lib().ag_sift_describe(L.ptr(P), 1, PS, C.c_float(0.2), L.ptr(out), L.stream_ptr()) != 0
    assert L.lib().ag_last_error().decode() == ("ag_sift_describe: unsupported patch size: 16..65 with a 4 x 4 pooling grid "
                                                 "(not 17, 18, 23, 28, 38, 48, 58)")
    torch.cuda.synchronize()
    assert bool((out == SENT).all())


@pytest.mark.parametrize("PS", (16, 41))
def test_sift_pyr_bit_exact(L, PS):
    B, H_, W, cap = 2, 90, 110, 5
    plan, buf = pyramid(L, B, H_, W, 3)
    lafs, oc, lv = keypoints(B, cap, 11 + PS, plan)
    cnt = torch.tensor([3, cap], dtype=torch.int32, device=DEV)
    out = torch.full((B, cap, 128), SENT, device=DEV)
    dl, do, dv = device_keypoints(lafs, oc, lv)
    L.check(L.lib().ag_sift_describe_pyr(C.byref(plan), L.ptr(buf), L.ptr(dl), L.ptr(do), L.ptr(dv), L.ptr(cnt), cap, PS, C.c_float(0.2),
                                          L.ptr(out), L.stream_ptr()))
    got = out.cpu().numpy()
    gk, pk = sift_windows(L, PS)
    for b, n in ((0, 3), (1, cap)):
        assert (got[b, n:] == SENT).all()
        for i in range(n):
            P = H.sample(plane(plan, buf, b, oc[b, i], lv[b, i]), lafs[b, i:i + 1], PS)
            assert same(got[b, i], H.sift(P, gk, pk, 0.2, lambda y, x: probe(L, y, x)[0])[0]), (b, i)


# ---- the fused pyramid kernels ---------------------------------------------------------------------------------------------------------
def pyramid(L, B, H_, W, seed):
    plan = L.make_plan(B, H_, W, 3, 1.6, 5)
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(B, H_, W, generator=g) * 255).to(DEV)
    buf = torch.full((plan.total_floats,), SENT, device=DEV)
    L.check(L.lib().ag_pyramid_build(C.byref(plan), L.ptr(x), L.ptr(buf), L.stream_ptr()))
    torch.cuda.synchronize()
    return plan, buf


def plane(plan, buf, b, o, l):
    o = min(max(int(o), 0), plan.n_octaves - 1)
    l = min(max(int(l), 0), plan.n_levels - 1)
    n = plan.B * plan.h[o] * plan.w[o]
    off = plan.level_offset[o][l]
    return buf[off:off + n].view(plan.B, plan.h[o], plan.w[o])[b].cpu().numpy()


def device_keypoints(lafs, oc, lv):
    """The device copies of keypoints(); held by the caller for the whole call (a temporary inside the argument list could be freed,
    and its memory reused, before the kernel reads it)."""
    return dev(lafs), dev(oc, torch.int32), dev(lv, torch.int32)


def keypoints(B, cap, seed, plan):
    """Normalised LAFs [B,cap,2,3] (some partly outside the image), octave / level indices with out-of-range values (clamped)."""
    rng = np.random.default_rng(seed)
    A = (rng.random((B, cap, 2, 2)) - 0.5) * 0.3
    A[..., 0, 0] += 0.12; A[..., 1, 1] += 0.12
    lafs = np.concatenate([A, rng.random((B, cap, 2, 1)) * 1.2 - 0.1], axis=3).astype(np.float32)
    oc = rng.integers(-2, plan.n_octaves + 2, (B, cap)).astype(np.int32)
    lv = rng.integers(-2, plan.n_levels + 2, (B, cap)).astype(np.int32)
    return lafs, oc, lv


@pytest.mark.parametrize("PS", (3, 19, 41))
@pytest.mark.parametrize("B,counts", [(1, (6,)), (3, (0, -1, 4))], ids=["B1-full", "B3-zero-neg-partial"])
def test_orientation_hist_pyr_bit_exact(L, PS, B, counts):
    cap = 6
    plan, buf = pyramid(L, B, 80, 96, PS + B)
    lafs, oc, lv = keypoints(B, cap, PS * 7 + B, plan)
    out = torch.full((B, cap, 2, 2), SENT, device=DEV)
    gk = ori_gk(PS)
    dl, do, dv = device_keypoints(lafs, oc, lv)
    cnt = torch.tensor(counts, dtype=torch.int32, device=DEV)
    L.check(L.lib().ag_debug_orientation_hist_pyr(C.byref(plan), L.ptr(buf), L.ptr(dl), L.ptr(do), L.ptr(dv), L.ptr(cnt), cap, PS,
                                                   gk.ctypes.data_as(C.c_void_p), L.ptr(out), L.stream_ptr()))
    got = out.cpu().numpy()
    a2 = lambda y, x: probe(L, y, x)[0]      # noqa: E731
    cs = lambda x: probe(L, x, x)[1]         # noqa: E731
    sn = lambda x: probe(L, x, x)[2]         # noqa: E731
    for b, c in enumerate(counts):
        n = max(0, min(c, cap))
        assert (got[b, n:] == SENT).all(), (b, c)
        for i in range(n):
            R = H.orientation_hist_pyr(plane(plan, buf, b, oc[b, i], lv[b, i]), lafs[b, i:i + 1], PS, gk, a2, cs, sn)
            assert same(got[b, i], R[0]), (b, i, got[b, i], R[0])


@pytest.mark.parametrize("PS", (3, 19, 41))
@pytest.mark.parametrize("iters", (1, 2, 16))
@pytest.mark.parametrize("B,counts", [(1, (6,)), (3, (0, -1, 4))], ids=["B1-full", "B3-zero-neg-partial"])
def test_baumberg_pyr_bit_exact(L, PS, iters, B, counts):
    cap = 6
    plan, buf = pyramid(L, B, 80, 96, PS + iters + B)
    lafs, oc, lv = keypoints(B, cap, PS * 5 + iters + B, plan)
    out = torch.full((B, cap, 2, 2), SENT, device=DEV)
    gk = aff_gk(PS)
    dl, do, dv = device_keypoints(lafs, oc, lv)
    cnt = torch.tensor(counts, dtype=torch.int32, device=DEV)
    L.check(L.lib().ag_debug_baumberg_pyr(C.byref(plan), L.ptr(buf), L.ptr(dl), L.ptr(do), L.ptr(dv), L.ptr(cnt), cap, PS, iters,
                                           gk.ctypes.data_as(C.c_void_p), L.ptr(out), L.stream_ptr()))
    got = out.cpu().numpy()
    for b, c in enumerate(counts):
        n = max(0, min(c, cap))
        assert (got[b, n:] == SENT).all(), (b, c)
        for i in range(n):
            ref = H.baumberg_pyr(plane(plan, buf, b, oc[b, i], lv[b, i]), lafs[b, i:i + 1], PS, gk, iters)
            assert same(got[b, i], ref[0]), (b, i, got[b, i], ref[0])
