"""Generates tests/golden/given.npz by running the UNMODIFIED reference (/root/reference, ducha-aiki/affnet) on CPU, through the same
harness as make_golden.py (oracle/ref_harness.py).  Re-run only when the reference changes:

    python tests/golden/make_golden_given.py

Outputs (given.npz, compressed):
  ell_in, ell_lafs      ells2LAFsT (LAF.py:76-89) of the ellipses of ell.npz followed by synthetic ones: b = 0, near-circular, elongated,
                        rotated, and not positive definite (NaN in the reference)
  in_dLAFs              [n,2,3] upright pixel keypoints of the 256x320 graf crop: its plain detections (num_Baum_iters = 0, K = 300,
                        no orientation) followed by hand-placed keypoints near, on and across the image border
  src, out_dLAFs, desc  the reference's composition on in_dLAFs with the shipped AffNet / OriNet / HardNet++, as its
                        SIFT-AffNet-HardNet notebook chains the steps: pyramid of the detector's forward,
                        get_pyramid_and_level_index_for_LAFs(dLAFs, PS = 32), normalizeLAFs, getAffineShape(num_features = 0) with
                        num_Baum_iters = 1 (resp = the row index, so the kept responses are the source rows), getOrientation,
                        denormalizeLAFs, extract_patches_from_pyr(., 32) and HardNet
"""
import contextlib
import io
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
import ref_harness as R  # noqa: E402

warnings.filterwarnings("ignore")
torch.set_num_threads(8)


def quiet():
    return contextlib.redirect_stdout(io.StringIO())


def gray_of(rgb):
    return torch.from_numpy(np.mean(rgb, axis=2).astype(np.float32)).view(1, 1, rgb.shape[0], rgb.shape[1])


def synthetic_ells():
    rows = [
        (10.0, 20.0, 0.04, 0.0, 0.01),        # b = 0: the mask branch
        (5.5, 7.25, 0.01, 0.0, 0.01),         # circle, b = 0
        (100.0, 50.0, 0.02, 1e-7, 0.02),      # near-circular
        (30.0, 40.0, 0.0101, 0.0, 0.0099),
        (1.0, 2.0, 1.0, 0.0, 1e-4),           # elongated
        (3.0, 4.0, 1e-4, 0.0, 1.0),
        (7.0, 8.0, 0.5, 0.49, 0.5),           # elongated along the diagonal
        (9.0, 1.0, 0.03, -0.01, 0.02),        # rotated
        (11.0, 12.0, 0.02, 0.015, 0.04),
        (0.0, 0.0, 2.0, -1.5, 3.0),
        (13.0, 14.0, 0.01, 0.02, 0.01),       # a c < b^2: not positive definite
        (15.0, 16.0, -0.01, 0.0, 0.02),       # a < 0
        (17.0, 18.0, 0.0, 0.0, 0.0),          # degenerate
    ]
    g = torch.Generator().manual_seed(41)
    ang = torch.rand(24, generator=g) * 6.283185307179586
    s1 = torch.exp(torch.rand(24, generator=g) * 6.0 - 3.0)
    s2 = s1 * torch.exp(torch.rand(24, generator=g) * 3.0)
    for t, l1, l2 in zip(ang.tolist(), (1.0 / s1 ** 2).tolist(), (1.0 / s2 ** 2).tolist()):
        c, s = np.cos(t), np.sin(t)
        rows.append((float(np.float32(t * 17.0)), float(np.float32(t * 5.0)), c * c * l1 + s * s * l2, c * s * (l1 - l2), s * s * l1 + c * c * l2))
    return torch.tensor(rows, dtype=torch.float32)


def hand_placed(H, W):
    """Upright keypoints (x, y, s) -> [[s, 0, x], [0, s, y]]: inside, touching, on and across each border, and outside the image."""
    pts = [(W / 2.0, H / 2.0, 20.0), (25.0, 30.0, 12.0), (12.0, 100.0, 12.0), (W - 12.0, 120.0, 12.0), (3.0, 60.0, 9.0),
           (W - 1.0, 80.0, 6.0), (150.0, 2.0, 10.0), (160.0, H - 4.0, 8.0), (-6.0, 50.0, 5.0), (W + 10.0, 90.0, 7.0),
           (100.0, -20.0, 15.0), (0.0, 0.0, 4.0), (W - 40.0, H - 40.0, 39.0), (200.0, 150.0, 60.0), (64.0, 64.0, 2.5),
           (180.0, 70.0, 30.0)]
    out = torch.zeros(len(pts), 2, 3)
    for i, (x, y, s) in enumerate(pts):
        out[i, 0, 0], out[i, 1, 1], out[i, 0, 2], out[i, 1, 2] = s, s, x, y
    return out


def main():
    m = R.ref_modules()
    LAF, SIR = m["LAF"], m["SparseImgRepresenter"]
    aff, ori, hn = R.load_nets()
    out = {}
    ell = torch.from_numpy(np.load(os.path.join(HERE, "ell.npz"))["ell"]).float()
    out["ell_in"] = torch.cat([ell, synthetic_ells()], dim=0)
    with torch.no_grad():
        out["ell_lafs"] = LAF.ells2LAFsT(out["ell_in"])

    img = gray_of(np.load(os.path.join(HERE, "graf_crop.npz"))["rgb"])
    H, W = img.size(2), img.size(3)
    kw = dict(mrSize=5.192, num_features=300, border=5, AffNet=aff, OriNet=ori)
    det0 = SIR.ScaleSpaceAffinePatchExtractor(num_Baum_iters=0, **kw)
    det1 = SIR.ScaleSpaceAffinePatchExtractor(num_Baum_iters=1, **kw)
    with torch.no_grad(), quiet():
        plain, _ = det0(img, do_ori=False)                      # the detector's forward also builds the pyramid
        dL = torch.cat([plain, hand_placed(H, W)], dim=0)
        det1.scale_pyr, det1.sigmas, det1.pix_dists = det0.scale_pyr, det0.sigmas, det0.pix_dists
        pidx, lidx = LAF.get_pyramid_and_level_index_for_LAFs(dL, det1.sigmas, det1.pix_dists, 32)
        nL = LAF.normalizeLAFs(dL, W, H)
        resp = torch.arange(dL.size(0)).float()
        r, L2, p2, l2 = det1.getAffineShape(resp, nL, pidx, lidx, num_features=0)
        L3 = det1.getOrientation(L2, p2, l2)
        dL3 = LAF.denormalizeLAFs(L3, W, H)
        desc = hn(det1.extract_patches_from_pyr(dL3, PS=32))
    out.update(in_dLAFs=dL, src=r.long(), out_dLAFs=dL3, desc=desc, n_plain=plain.size(0))
    path = os.path.join(HERE, "given.npz")
    np.savez_compressed(path, **{k: (v.detach().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in out.items()})
    print("given.npz %.1f KB: %d ellipses, %d keypoints in (%d detected), %d survivors" % (
        os.path.getsize(path) / 1024.0, out["ell_in"].size(0), dL.size(0), plain.size(0), dL3.size(0)))


if __name__ == "__main__":
    main()
