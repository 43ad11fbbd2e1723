"""Given keypoints, restated: ells2LAFsT (LAF.py:76-89) as numpy fp32 operations one by one, the arithmetic of ag_ells_to_lafs, and the
reference's composition on caller-supplied pixel LAFs - get_pyramid_and_level_index_for_LAFs(dLAFs, 32), normalizeLAFs, getAffineShape's
keep-all branch, getOrientation, denormalizeLAFs and extract_patches_from_pyr + descriptor - built from the oracle's stages.
tests/golden/given.npz pins both to the unmodified reference (tests/test_given_cpu.py)."""
import numpy as np
import torch

import affnet_oracle as O
import oracle_estimators as OE

f32 = np.float32


def _sign(x):
    """torch.sign: (x > 0) - (x < 0), so 0 for +-0 and NaN."""
    return (x > 0).astype(f32) - (x < 0).astype(f32)


def _rectify(a00, a01, a10, a11):
    """rectifyAffineTransformationUpIsUp (LAF.py:285-291) -> (A00, A01, A10, A11)."""
    det = np.sqrt(np.abs(a00 * a11 - a10 * a01 + f32(1e-10)))
    b2a2 = np.sqrt(a01 * a01 + a00 * a00)
    return b2a2 / det, f32(0) * det, (a11 * a01 + a10 * a00) / (b2a2 * det), det / b2a2


def ells_to_lafs(ells):
    """[n,5] (x, y, a, b, c) -> [n,2,3] float32, each torch operation of ells2LAFsT / invSqrtTorch one fp32 operation."""
    e = np.asarray(ells, dtype=f32).reshape(-1, 5)
    a, b, c = e[:, 2], e[:, 3], e[:, 4]
    with np.errstate(all="ignore"):
        sc = np.sqrt(np.sqrt(a * c - b * b + f32(1e-12)))
        mask = (b != 0).astype(f32)
        r1 = mask * (c - a) / (f32(2.0) * b + f32(1e-12))
        t1 = _sign(r1) / (np.abs(r1) + np.sqrt(f32(1.0) + r1 * r1))
        r = f32(1.0) / np.sqrt(f32(1.0) + t1 * t1)
        t = t1 * r
        r = r * mask + f32(1.0) * (f32(1.0) - mask)
        t = t * mask
        x = f32(1.0) / np.sqrt(r * r * a - f32(2.0) * r * t * b + t * t * c)
        z = f32(1.0) / np.sqrt(t * t * a + f32(2.0) * r * t * b + r * r * c)
        d = np.sqrt(x * z)
        x = x / d
        z = z / d
        ia = r * r * x + t * t * z
        ib = -r * t * x + t * r * z
        ic = t * t * x + r * r * z
        a00, a01, a11 = ia / sc, ib / sc, ic / sc
        s = np.sqrt(np.abs(a00 * a11 - a01 * a01))
        R = _rectify(a00 / s, a01 / s, a01 / s, a11 / s)
        out = np.zeros((len(e), 2, 3), dtype=f32)
        out[:, 0, 0], out[:, 0, 1], out[:, 1, 0], out[:, 1, 1] = R[0] * s, R[1] * s, R[2] * s, R[3] * s
    out[:, 0, 2], out[:, 1, 2] = e[:, 0], e[:, 1]
    return out


def knife_edge(A, rel=64.0):
    """Rows whose batch_eig2x2 discriminant trace^2 - 4 det is within fp32 rounding of zero: its sign decides between the eigenvalues
    and the (1000, 1e-4) fallback, so the last bits of A decide the eigenvalue-ratio test.  An upright keypoint whose AffNet shape is
    nearly isotropic lands there."""
    tr = A[:, 0, 0] + A[:, 1, 1]
    det = A[:, 0, 0] * A[:, 1, 1] - A[:, 1, 0] * A[:, 0, 1]
    return (tr * tr - 4 * det).abs() <= rel * float(np.finfo(np.float32).eps) * tr * tr


def describe_given(x, dLAFs, shape="affnet", num_iters=1, aff_sd=None, ori=None, ori_sd=None, hard_sd=None, sift_ps=None, border=5, nlevels=3,
                   init_sigma=1.6, shape_ps=19, ori_ps=19):
    """The reference's steps on caller-supplied pixel LAFs dLAFs [n,2,3] of image x [1,1,H,W]: shape "affnet" (aff_sd) / "baumberg" / None
    with num_iters iterations and the keep-all filter, ori "orinet" (ori_sd) / "histogram" / None, then HardNet (hard_sd) or, with
    sift_ps, SIFTNet(sift_ps).  Every estimator samples the level get_pyramid_and_level_index_for_LAFs(dLAFs, 32) picks.
    Returns (dLAFs out [m,2,3] px, src [m] input rows, desc [m,128], state).  With neither step the LAFs are the input ones."""
    pyr, sigmas, pix = O.scale_pyramid(x, nlevels, init_sigma, border)
    pidx, lidx = O.pyramid_level_for_lafs(dLAFs, sigmas, pix, 32)
    LAFs = O.normalize_lafs(dLAFs, x.size(3), x.size(2))
    src = torch.arange(dLAFs.size(0))
    shaped = shape is not None and num_iters > 0
    dbg = {}
    if shaped:
        if shape == "affnet":
            est, PS = (lambda P: O.affnet_forward(P, aff_sd)), 32
        elif shape == "baumberg":
            est, PS = O.baumberg_shape, shape_ps
        else:
            raise ValueError("shape: affnet, baumberg or None")
        resp = src.float()
        _, LAFs, pidx, lidx, dbg["aff"] = OE.get_affine_shape_iter(pyr, resp, LAFs, pidx, lidx, -1, est, num_iters, PS)
        src = dbg["aff"]["idxs"]
    if ori == "orinet":
        LAFs, dbg["ori"] = O.get_orientation(pyr, LAFs, pidx, lidx, ori_sd)
    elif ori == "histogram":
        patches = O.extract_patches_from_pyramid(pyr, pidx, lidx, LAFs, ori_ps)
        LAFs = torch.cat([torch.bmm(LAFs[:, :, :2], OE.angles2A(O.orientation_hist(patches))), LAFs[:, :, 2:]], dim=2)
    elif ori is not None:
        raise ValueError("ori: orinet, histogram or None")
    out = O.denormalize_lafs(LAFs, x.size(3), x.size(2)) if (shaped or ori is not None) else dLAFs.clone()
    state = dict(pyr=pyr, sigmas=sigmas, pix_dists=pix, pyr_idxs=pidx, level_idxs=lidx, debug=dbg)
    if sift_ps is not None:
        import oracle_sift as OS
        desc, _, _ = OS.describe_sift(out, state, sift_ps)
    else:
        desc, _, _ = O.describe(out, state, hard_sd)
    return out, src, desc, state
