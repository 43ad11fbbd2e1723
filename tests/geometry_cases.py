"""Constructed inputs for the keypoint-geometry tests (tests/test_geometry_cpu.py, tests/test_gpu_geometry.py).

Every set is deterministic (fixed seeds, or searches over consecutive floats) and float32.  The searches use the restatement
(tests/geometry_restated.py) only to place a value exactly where a test needs it: on a boundary, one ulp from it, or where two fp32
evaluation orders disagree."""
import functools

import numpy as np

import geometry_restated as G

F = np.float32
A_EXACT = np.array([[2, 0], [0, 1]], np.float32)   # a power-of-two diagonal: the compose is exact and passes the eigen test (ratio 2)


def ulps(x, k):
    """The float k ulps from fp32 x (k may be an array)."""
    return (np.asarray(x, np.float32).view(np.int32) + np.asarray(k, np.int32)).view(np.float32)


def _lafs_for_exact_A(NL):
    """Detector LAFs that A_EXACT composes into NL exactly (row 0 of the A part halves, row 1 stays)."""
    L = G.f32(NL).copy()
    L[:, 0, :2] = L[:, 0, :2] / F(2)
    return L


# ---- boundary ------------------------------------------------------------------------------------------------------------------
SAFE_ROW = (F(1 / 16), F(1 / 32), F(0.5))          # corners 0.5 +- 3/32: far inside


def boundary_exact():
    """A corner coordinate exactly at 0 or 1, or at the nearest value on either side that the row can reach exactly (+-2^-26 around 0,
    the fp32 neighbours of 1), for each corner, in the x and the y row.  Every sum is exact, so both summation orders give the same
    corners and only the inclusive comparisons are tested.  -> (A [n,2,2], L [n,2,3], keep [n]): keep is what they must decide."""
    NL, keep = [], []
    for row in (0, 1):
        for (x, y) in G.CORNERS:
            for T in (0.0, 1.0):
                # the target corner is the row's minimum (T = 0) or maximum (T = 1); the other corners stay inside
                s = -1.0 if T == 0.0 else 1.0
                h0, h1 = F(s * x / 8), F(s * y / 16)
                for k in (-1, 0, 1):
                    corner = k * 2.0 ** -26 if T == 0.0 else float(ulps(F(1), k))
                    h2 = corner - (float(h0) * x + float(h1) * y)
                    assert float(F(h2)) == h2
                    r = np.zeros((2, 3), np.float32)
                    r[row] = (h0, h1, h2)
                    r[1 - row] = SAFE_ROW
                    NL.append(r)
                    keep.append(k == 0 or (k > 0) == (T == 0.0))
    NL = np.stack(NL)
    return np.broadcast_to(A_EXACT, (len(NL), 2, 2)).copy(), _lafs_for_exact_A(NL), np.array(keep)


def corner_fused_order(NL):
    """The corners summed as h0*x + (h1*y + h2) (the other association): -> [n,2,4]."""
    NL = G.f32(NL)
    out = np.empty((NL.shape[0], 2, 4), np.float32)
    for c, (x, y) in enumerate(G.CORNERS):
        out[:, :, c] = NL[:, :, 0] * F(x) + (NL[:, :, 1] * F(y) + NL[:, :, 2])
    return out


@functools.lru_cache(maxsize=None)
def boundary_association(n_each=12, seed=5):
    """Rows whose corner sum lands on opposite sides of 0 or of 1 under (h0*x + h1*y) + h2 and h0*x + (h1*y + h2), in the x row and in
    the y row, for each of the four corners.  -> (A, L): A is A_EXACT, so the composed LAF is exactly the constructed one."""
    g = np.random.default_rng(seed)
    NL = []
    for row in (0, 1):
        for ci, (x, y) in enumerate(G.CORNERS):
            for T in (0.0, 1.0):
                s = -1.0 if T == 0.0 else 1.0
                m = 200000
                h0 = (g.uniform(0.02, 0.2, m) * s * x).astype(np.float32)
                h1 = (g.uniform(0.02, 0.2, m) * s * y).astype(np.float32)
                base = F(T) - (h0 * F(x) + h1 * F(y))
                h2 = ulps(base, g.integers(-2, 3, m))
                cand = np.zeros((m, 2, 3), np.float32)
                cand[:, row, 0], cand[:, row, 1], cand[:, row, 2] = h0, h1, h2
                cand[:, 1 - row] = SAFE_ROW
                a, b = G.corners(cand)[:, row, ci], corner_fused_order(cand)[:, row, ci]
                flip = ((a < 0) != (b < 0)) if T == 0.0 else ((a > 1) != (b > 1))
                idx = np.nonzero(flip)[0][:n_each]
                assert len(idx) == n_each, (row, ci, T, len(idx))
                NL.append(cand[idx])
    NL = np.concatenate(NL)
    return np.broadcast_to(A_EXACT, (len(NL), 2, 2)).copy(), _lafs_for_exact_A(NL)


# ---- eigen-ratio -------------------------------------------------------------------------------------------------------------
EIGEN_LAF = np.array([[0.01, 0.0, 0.5], [0.0, 0.01, 0.5]], np.float32)   # composed with any finite A of the set it stays inside


@functools.lru_cache(maxsize=None)
def ratio_neighbours():
    """Diagonal A whose ratio |l1 / (l2 + 1e-8)| is exactly 6 or fp32(1/6), or the float on either side: {ratio: A}."""
    targets = {float(ulps(v, k)) for v in (F(6), G.SIXTH) for k in (-1, 0, 1)}
    found = {}
    for b in (1, 0.5, 0.75, 1.25, 3, 0.1, 0.3, 2.5, 7):
        b = F(b)
        for neg in (False, True):
            cand = ulps(F(-6) * b if neg else F(6) * b, np.arange(-64, 65))
            A = np.zeros((len(cand), 2, 2), np.float32)
            A[:, 0, 0], A[:, 1, 1] = (b, cand) if neg else (cand, b)
            for a, r in zip(A, G.eig_ratio(A)):
                if float(r) in targets:
                    found.setdefault(float(r), a)
    assert len(found) == len(targets), sorted(found)
    return found


def eigen_cases():
    """-> (A [n,2,2], L [n,2,3], names): the ratio's neighbours of 6 and 1/6, delta1 = 0 and < 0, l2 = -1e-8 (ratio inf), negative
    ratios, det <= 0, A = 0, inf and NaN in A, and NaN / inf in the LAF under a good A."""
    t = F(1e-8)
    named = [("ratio %.9g" % r, a) for r, a in sorted(ratio_neighbours().items())]
    named += [
        ("identity (delta1 = 0)", [[1, 0], [0, 1]]), ("2I (delta1 = 0)", [[2, 0], [0, 2]]),
        ("rotation 90 (delta1 < 0)", [[0, -1], [1, 0]]), ("similarity (delta1 < 0)", [[1, -1], [1, 1]]),
        ("l2 = -1e-8 (ratio inf)", [[0, t], [t, 0]]),
        ("det < 0, l = 1, -2", [[1, 0], [0, -2]]), ("det < 0, l = -2, 1", [[-2, 0], [0, 1]]), ("det < 0, l = -6, 1", [[-6, 0], [0, 1]]),
        ("both negative, ratio 1/3", [[-1, 0], [0, -3]]), ("det = 0", [[1, 0], [0, 0]]), ("det = 0, rank 1", [[1, 2], [2, 4]]),
        ("A = 0", [[0, 0], [0, 0]]), ("A inf", [[np.inf, 0], [0, 1]]), ("A -inf off-diagonal", [[1, -np.inf], [0, 1]]),
        ("A NaN", [[np.nan, 0], [0, 1]]), ("A NaN off-diagonal", [[1, 0], [np.nan, 1]]), ("shear 1.5", [[1, 1.5], [0, 1]]),
    ]
    A = np.array([np.asarray(a, np.float32) for _, a in named], np.float32)
    L = np.broadcast_to(EIGEN_LAF, (len(A), 2, 3)).copy()
    names = [n for n, _ in named]
    bad = [("LAF NaN centre", [[0.01, 0, np.nan], [0, 0.01, 0.5]]), ("LAF NaN shape", [[np.nan, 0, 0.5], [0, 0.01, 0.5]]),
           ("LAF inf centre", [[0.01, 0, np.inf], [0, 0.01, 0.5]]), ("LAF -inf shape", [[0.01, 0, 0.5], [0, -np.inf, 0.5]])]
    A = np.concatenate([A, np.broadcast_to(A_EXACT, (len(bad), 2, 2))])
    L = np.concatenate([L, np.array([np.asarray(l, np.float32) for _, l in bad], np.float32)])
    return A, L, names + [n for n, _ in bad]


# ---- responses -------------------------------------------------------------------------------------------------------------------
def response_case():
    """One image whose top-K cut runs through tied zeros: survivors with negative, -0.0 and tied positive responses, and rejected rows
    (identity A fails the eigen test) with positive, negative and -0.0 responses.  With num_features in RESPONSE_NF the reference's
    resp * mask puts rejected rows (as zeros) ahead of the negative survivors.  -> (A, L, resp, keep)."""
    keep = np.array([1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1], bool)
    resp = np.array([-0.5, 0.3, -0.25, 0.75, -0.2, -0.0, 0.75, 5.0, -1.0, 0.0, -0.0, 0.125], np.float32)
    A = np.where(keep[:, None, None], A_EXACT, np.eye(2, dtype=np.float32)).astype(np.float32)
    L = np.broadcast_to(EIGEN_LAF, (len(keep), 2, 3)).copy()
    return A, L, resp, keep


RESPONSE_NF = (1, 2, 3, 4, 5, 6, 7, 8)


# ---- random rows ---------------------------------------------------------------------------------------------------------------
def random_A(n, seed, max_aniso=9.0):
    """Affine shapes R(t) diag(s a, s / a) R(p) with full mantissas: a in [1, sqrt(max_aniso)], so the eigen test keeps part of them."""
    g = np.random.default_rng(seed)
    t = g.uniform(-np.pi, np.pi, n)
    p = -t + g.uniform(-0.4, 0.4, n)                # near-symmetric, so the eigenvalues are mostly real
    a = np.sqrt(g.uniform(1.0, max_aniso, n)); s = g.uniform(0.5, 2.0, n)
    rot = lambda q: np.stack([np.stack([np.cos(q), -np.sin(q)], -1), np.stack([np.sin(q), np.cos(q)], -1)], -2)  # noqa: E731
    D = np.zeros((n, 2, 2)); D[:, 0, 0] = s * a; D[:, 1, 1] = s / a
    return (rot(t) @ D @ rot(p)).astype(np.float32)


def random_lafs(n, seed, lo=0.005, hi=0.3):
    """Normalised detector LAFs: centres in [0.02, 0.98], isotropic A parts of scale [lo, hi] with random off-diagonal noise, so a
    good share of them touches the boundary after the compose."""
    g = np.random.default_rng(seed)
    L = np.zeros((n, 2, 3))
    sc = g.uniform(lo, hi, n)
    L[:, 0, 0] = sc * g.uniform(0.8, 1.2, n); L[:, 1, 1] = sc * g.uniform(0.8, 1.2, n)
    L[:, 0, 1] = sc * g.uniform(-0.3, 0.3, n); L[:, 1, 0] = sc * g.uniform(-0.3, 0.3, n)
    L[:, :, 2] = g.uniform(0.02, 0.98, (n, 2))
    return L.astype(np.float32)


def random_resp(n, seed, levels=64):
    """Responses with many ties (quantised to `levels` values), zeros, negatives and -0.0."""
    g = np.random.default_rng(seed)
    r = (np.floor(g.uniform(-0.2, 1.0, n) * levels) / levels).astype(np.float32)
    r[g.random(n) < 0.05] = F(-0.0)
    return r


def random_full(n, seed, lo=-4.0, hi=4.0):
    """Full-mantissa entries for the 2x2 products: about a quarter of the fused products differ from the unfused ones."""
    return np.random.default_rng(seed).uniform(lo, hi, n).astype(np.float32)


def shape_rows(n, seed):
    """n rows (A, L, resp) for the shape filter: the constructed boundary, association and eigen rows first (as many as fit), random
    rows after them."""
    Ab, Lb, _ = boundary_exact()
    Aa, La = boundary_association()
    Ae, Le, _ = eigen_cases()
    A = np.concatenate([Ab, Aa, Ae, random_A(n, seed)])[:n]
    L = np.concatenate([Lb, La, Le, random_lafs(n, seed + 1)])[:n]
    return np.ascontiguousarray(A), np.ascontiguousarray(L), random_resp(n, seed + 2)


# ---- ellipses --------------------------------------------------------------------------------------------------------------------
def ell_cases(seed=11):
    """Pixel LAFs for LAFs2ellT: isotropic and near-isotropic, anisotropy (singular-value ratio) up to 1e3, rotations at multiples of
    pi/4, det < 0, and the zero LAF.  -> (L [n,2,3], elongation [n] in float64; inf where the LAF is singular)."""
    g = np.random.default_rng(seed)
    rows = []
    for aniso in (1.0, 1.0 + 1e-6, 1.0 + 1e-3, 1.5, 6.0, 30.0, 1e2, 1e3):
        for k in range(8):
            for s in (0.5, 3.0, 40.0):
                q, p = k * np.pi / 4, g.uniform(-np.pi, np.pi)
                R = lambda a: np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])  # noqa: E731
                A = s * (R(q) @ np.diag([np.sqrt(aniso), 1 / np.sqrt(aniso)]) @ R(p))
                rows.append(np.concatenate([A, g.uniform(0, 500, (2, 1))], 1))
    for k in range(8):                                       # exactly isotropic rotations, no noise
        q = k * np.pi / 4
        rows.append(np.array([[5 * np.cos(q), -5 * np.sin(q), 10.0], [5 * np.sin(q), 5 * np.cos(q), 20.0]]))
    rows += [np.array([[3.0, 0, 1], [0, -2, 2]]), np.array([[0, 2.0, 1], [2, 0, 2]]), np.array([[-1.0, 0.5, 7], [0.3, 4, 8]]),
             np.zeros((2, 3))]
    L = np.array(rows).astype(np.float32)
    sv = np.linalg.svd(L[:, :, :2].astype(np.float64), compute_uv=False)
    with np.errstate(divide="ignore", invalid="ignore"):
        elong = sv[:, 0] / sv[:, 1]
    return L, np.where(np.isfinite(elong), elong, np.inf)
