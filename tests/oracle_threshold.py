"""ScaleSpaceAffinePatchExtractor.forward in the reference's threshold mode (th set, SparseImgRepresenter.py:33-37, 104-110, 151-156,
192-195), restated from the oracle's stages: the detector with th and num_features = -1 keeps every candidate of the accepted levels in
(octave, level, raster) order, and the shape step keeps every survivor in index order.  tests/golden/threshold.npz pins it to the
unmodified reference (tests/test_threshold_cpu.py)."""
import torch

import affnet_oracle as O
import oracle_estimators as OE


def detect(x, th, shape="affnet", num_iters=1, aff_sd=None, ori=None, ori_sd=None, border=5, mrSize=5.192, nlevels=3, init_sigma=1.6,
           shape_ps=19, ori_ps=19):
    """-> (dLAFs [N,2,3] px, responses [N], state) as oracle_estimators.detect, with threshold th and no top-K anywhere."""
    pyr, sigmas, pix = O.scale_pyramid(x, nlevels, init_sigma, border)
    resp, LAFs, pidx, lidx = O.multi_scale_detector(pyr, sigmas, -1, mrSize, th=th)
    LAFs = LAFs.clone()
    LAFs[:, 0:2, 0:2] = mrSize * LAFs[:, :, 0:2]
    dbg = dict(det_resp=resp.clone(), det_LAFs=LAFs.clone(), det_pidx=pidx.clone(), det_lidx=lidx.clone())
    if shape is not None and num_iters > 0:
        if shape == "affnet":
            est, PS = (lambda P: O.affnet_forward(P, aff_sd)), 32
        elif shape == "baumberg":
            est, PS = O.baumberg_shape, shape_ps
        else:
            raise ValueError("shape: affnet, baumberg or None")
        resp, LAFs, pidx, lidx, dbg["aff"] = OE.get_affine_shape_iter(pyr, resp, LAFs, pidx, lidx, -1, est, num_iters, PS)
    if ori == "orinet":
        LAFs, dbg["ori"] = O.get_orientation(pyr, LAFs, pidx, lidx, ori_sd)
    elif ori == "histogram":
        patches = O.extract_patches_from_pyramid(pyr, pidx, lidx, LAFs, ori_ps)
        R = OE.angles2A(O.orientation_hist(patches))
        LAFs = torch.cat([torch.bmm(LAFs[:, :, :2], R), LAFs[:, :, 2:]], dim=2)
        dbg["ori"] = dict(patches=patches, R=R)
    elif ori is not None:
        raise ValueError("ori: orinet, histogram or None")
    dLAFs = O.denormalize_lafs(LAFs, x.size(3), x.size(2))
    return dLAFs, resp, dict(pyr=pyr, sigmas=sigmas, pix_dists=pix, pyr_idxs=pidx, level_idxs=lidx, debug=dbg)
