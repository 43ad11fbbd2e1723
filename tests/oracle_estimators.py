"""CPU oracle for every estimator configuration of ScaleSpaceAffinePatchExtractor.forward (SparseImgRepresenter.py:189-209):
the loop of getAffineShape (SparseImgRepresenter.py:127-162) with AffNet or the Baumberg step (AffineShapeEstimator) and any
number of iterations, num_Baum_iters = 0 (no shape step), then OriNet, gradient-histogram or no orientation.

TEST INFRASTRUCTURE, NOT PRODUCT, built on oracle/affnet_oracle.py (whose `detect` is the AffNet x 1 case).  The reference's
own loop cannot pin the iterated configurations: under python 3 it raises TypeError at Utils.py:54.  So the Baumberg module is
pinned by tests/golden/handcrafted.npz, AffNet x 1 by affnet_oracle.get_affine_shape, and num_Baum_iters = 0 with the histogram
by the reference default detector's golden output (handcrafted.npz `default_dLAFs`); tests/test_pipeline_estimators_cpu.py
checks all three.
"""
import torch

import affnet_oracle as O


def angles2A(ang):
    """LAF.py:306-311: [[cos, sin], [-sin, cos]]."""
    c, s = torch.cos(ang).view(-1, 1, 1), torch.sin(ang).view(-1, 1, 1)
    return torch.cat([torch.cat([c, s], dim=2), torch.cat([-s, c], dim=2)], dim=1)


def _fma32(a, b, c):
    """fp32 fused multiply-add: the float64 product of two fp32 values is exact, so one rounding of the sum to fp32 (via float64; a
    double rounding differs from a single one only in rare ties)."""
    return (a.double() * b.double() + c.double()).float()


def extract_patches_fp32(img, LAFs, PS):
    """The CUDA sampler's fp32 arithmetic (common.cuh: laf_sample_xy + bilinear_zero, explicit roundings and fmas) restated in torch:
    the same closed form as affnet_oracle.extract_patches, which evaluates it in float64.  Used as an fp32-level perturbation of the
    oracle (conditioning of the iterated Baumberg loop, `shape_spread`)."""
    h, w = img.size(2), img.size(3)
    n = LAFs.size(0)
    Lf = LAFs.float()
    f = lambda v: torch.tensor(float(v), dtype=torch.float32)  # noqa: E731
    ms = f(min(h, w))
    col = lambda t: t.view(n, 1, 1).expand(n, PS, PS)  # noqa: E731
    a11, a12, tx = col(Lf[:, 0, 0] * ms), col(Lf[:, 0, 1] * ms), col(Lf[:, 0, 2] * f(w))
    a21, a22, ty = col(Lf[:, 1, 0] * ms), col(Lf[:, 1, 1] * ms), col(Lf[:, 1, 2] * f(h))
    j = torch.arange(PS, dtype=torch.float32)
    g = _fma32(torch.full_like(j, 2.0), j, torch.ones_like(j)) * (f(1.0) / f(PS)) - 1.0
    xj, yi = g.view(1, 1, PS).expand(n, PS, PS), g.view(1, PS, 1).expand(n, PS, PS)
    px = _fma32(a11, xj, _fma32(a12, yi, tx)) - 0.5
    py = _fma32(a21, xj, _fma32(a22, yi, ty)) - 0.5
    x0, y0 = torch.floor(px), torch.floor(py)
    ax, ay = px - x0, py - y0
    im = img.view(h, w).float()

    def tap(yy, xx):
        ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        v = im[yy.clamp(0, h - 1).long(), xx.clamp(0, w - 1).long()]
        return torch.where(ok, v, torch.zeros_like(v))

    top = _fma32(tap(y0, x0 + 1), ax, tap(y0, x0) * (1.0 - ax))
    bot = _fma32(tap(y0 + 1, x0 + 1), ax, tap(y0 + 1, x0) * (1.0 - ax))
    return _fma32(bot, ay, top * (1.0 - ay)).view(n, 1, PS, PS)


def extract_patches_from_pyramid_fp32(pyr, pyr_idxs, level_idxs, LAFs, PS=32):
    """affnet_oracle.extract_patches_from_pyramid with the CUDA sampler's fp32 arithmetic (extract_patches_fp32)."""
    out = torch.zeros(LAFs.size(0), 1, PS, PS)
    for o in range(len(pyr)):
        for l in range(len(pyr[o])):
            sel = ((pyr_idxs == o) & (level_idxs == l)).nonzero().view(-1)
            if sel.numel():
                out[sel] = extract_patches_fp32(pyr[o][l], LAFs[sel], PS)
    return out


def get_affine_shape_iter(pyr, resp, LAFs, pyr_idxs, level_idxs, num_features, estimator, num_iters, PS,
                          sampler=O.extract_patches_from_pyramid):
    """SparseImgRepresenter.py:127-162: `num_iters` (>= 1) iterations of `estimator` (patches [n,1,PS,PS] -> A [n,2,2]) sampled at
    the working LAFs of the original pyramid levels, base_A <- A base_A (the first iteration takes A as is: bmm(A, I) = A), then the
    eigen-ratio / boundary filter and the top-num_features selection of affnet_oracle.get_affine_shape."""
    base_A, cur, patches = None, LAFs, None
    for i in range(num_iters):
        patches = sampler(pyr, pyr_idxs, level_idxs, cur, PS)
        A = estimator(patches)
        base_A = A if base_A is None else torch.bmm(A, base_A)
        if i != num_iters - 1:
            cur = torch.cat([torch.bmm(base_A, LAFs[:, :, 0:2]), LAFs[:, :, 2:]], dim=2)
    new_LAFs = torch.cat([torch.bmm(base_A, LAFs[:, :, 0:2]), LAFs[:, :, 2:]], dim=2)
    mask = O.shape_filter_mask(base_A, new_LAFs)
    n_ok = int(mask.sum().item())
    if num_features > 0 and n_ok > num_features:
        r, idxs = torch.topk(resp * mask.float(), k=num_features)
    else:
        idxs = mask.nonzero().view(-1)
        r = resp[idxs]
    out_LAFs = torch.cat([torch.bmm(base_A[idxs], LAFs[idxs][:, :, 0:2]), LAFs[idxs][:, :, 2:]], dim=2)
    return r, out_LAFs, pyr_idxs[idxs], level_idxs[idxs], dict(patches=patches, A=A, base_A=base_A, mask=mask, idxs=idxs)


def detect(x, shape="affnet", num_iters=1, aff_sd=None, ori=None, ori_sd=None, num_features=2000, border=5, mrSize=5.192, nlevels=3,
           init_sigma=1.6, shape_ps=19, ori_ps=19):
    """ScaleSpaceAffinePatchExtractor.forward, th=None.  shape: "affnet" (aff_sd), "baumberg" (AffineShapeEstimator(shape_ps)) or None;
    num_iters = num_Baum_iters (0 = no shape step whatever `shape` says).  ori: "orinet" (ori_sd), "histogram" (OrientationDetector(ori_ps))
    or None.  Returns (dLAFs [N,2,3] px, responses [N], state) like affnet_oracle.detect; state["debug"] holds the stages' tensors."""
    pyr, sigmas, pix = O.scale_pyramid(x, nlevels, init_sigma, border)
    shaped = shape is not None and num_iters > 0
    pre = int(1.5 * num_features) if shaped else num_features           # SparseImgRepresenter.py:192-194
    resp, LAFs, pidx, lidx = O.multi_scale_detector(pyr, sigmas, pre, mrSize)
    LAFs = LAFs.clone()
    LAFs[:, 0:2, 0:2] = mrSize * LAFs[:, :, 0:2]
    dbg = dict(det_resp=resp.clone(), det_LAFs=LAFs.clone(), det_pidx=pidx.clone(), det_lidx=lidx.clone())
    if shaped:
        if shape == "affnet":
            est, PS = (lambda P: O.affnet_forward(P, aff_sd)), 32
        elif shape == "baumberg":
            est, PS = O.baumberg_shape, shape_ps
        else:
            raise ValueError("shape: affnet, baumberg or None")
        resp, LAFs, pidx, lidx, dbg["aff"] = get_affine_shape_iter(pyr, resp, LAFs, pidx, lidx, num_features, est, num_iters, PS)
    if ori == "orinet":
        LAFs, dbg["ori"] = O.get_orientation(pyr, LAFs, pidx, lidx, ori_sd)
    elif ori == "histogram":                                                   # SparseImgRepresenter.py:167-180, OriNet=OrientationDetector
        patches = O.extract_patches_from_pyramid(pyr, pidx, lidx, LAFs, ori_ps)
        R = angles2A(O.orientation_hist(patches))
        LAFs = torch.cat([torch.bmm(LAFs[:, :, :2], R), LAFs[:, :, 2:]], dim=2)
        dbg["ori"] = dict(patches=patches, R=R)
    elif ori is not None:
        raise ValueError("ori: orinet, histogram or None")
    dLAFs = O.denormalize_lafs(LAFs, x.size(3), x.size(2))
    return dLAFs, resp, dict(pyr=pyr, sigmas=sigmas, pix_dists=pix, pyr_idxs=pidx, level_idxs=lidx, debug=dbg)


def _nudge(LAFs, toward):
    out = LAFs.clone()
    out[:, :, :2] = torch.nextafter(out[:, :, :2], torch.full_like(out[:, :, :2], toward))
    return out


def shape_spread(state, num_features, num_iters, PS=19):
    """Conditioning of the Baumberg loop of a `detect(shape="baumberg")` run (its `state`): the loop is re-run under four fp32-level
    perturbations - the CUDA sampler's fp32 arithmetic instead of the float64 sampler, a float64 Baumberg step (rounded to fp32), and
    the input LAFs' A moved by one ulp up / down - and for every prefilter row the largest change of base_A relative to its scale
    sqrt|det| is returned ([M], float64).  A keypoint whose base_A moves under such a perturbation cannot be expected to agree with
    another fp32 implementation (whose sampler and summation order differ by more than one ulp) any closer than that."""
    d = state["debug"]
    pyr, resp, LAFs, pidx, lidx = state["pyr"], d["det_resp"], d["det_LAFs"], d["det_pidx"], d["det_lidx"]

    def base_A(est=O.baumberg_shape, L0=LAFs, sampler=O.extract_patches_from_pyramid):
        return get_affine_shape_iter(pyr, resp, L0, pidx, lidx, num_features, est, num_iters, PS, sampler)[4]["base_A"].double()

    ref = base_A()
    s = (ref[:, 0, 0] * ref[:, 1, 1] - ref[:, 0, 1] * ref[:, 1, 0]).abs().sqrt()
    variants = [base_A(sampler=extract_patches_from_pyramid_fp32), base_A(est=lambda P: O.baumberg_shape(P.double())),
                base_A(L0=_nudge(LAFs, 1e9)), base_A(L0=_nudge(LAFs, -1e9))]
    return torch.stack([(ref - v).abs().amax(dim=(1, 2)) / s for v in variants]).amax(dim=0)
