"""ReprojectionStuff.py counterpart for verifying matches on the device: the reference's ground-truth checks
(get_GT_correspondence_indexes, ReprojectionStuff.py:126-137, and the affine-shape ones, get_GT_correspondence_indexes_Fro and
_Fro_and_center, :139-203, on tentatives or on whole detection sets), homography RANSAC (the notebook's ransac_validate) and
fundamental-matrix RANSAC (its findFundamentalMatrix alternative, also as DEGENSAC), for one pair or for every pair of a batch in one call.  The batched calls take DetectDescribePipeline.run's LAFs and
Losses.match_snn_pairs' (tent, ntent) as they are, never synchronise with the host, and are capturable in the same CUDA graph."""
import torch

from . import _lib as L

MAX_TCAP = 4194240   # ag_match_pairs' cap1 limit
# find_homography_pairs(affine=True)'s frame threshold: the smallest of {0.5, 1, 2, 4} (4 is the reference's threshold for this distance)
# that keeps >= 95 % of the GT-true tentatives of the warped pairs and graf 1->6 under the true H (DESIGN.md, profiles/affine_ransac_h100.json)
AFFINE_LAF_TH = 0.5


def _int_shape(t, shape, name, fn, label=None):
    if (not isinstance(t, torch.Tensor) or t.dim() != len(shape) or any(s is not None and t.size(k) != s for k, s in enumerate(shape))
            or t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool):
        raise L.AffnetB200Error("%s: %s must be an integer tensor [%s]" % (fn, name, label or ",".join(map(str, shape))))


def _lafs_shape(t, name, fn):
    if not isinstance(t, torch.Tensor) or t.dim() != 4 or tuple(t.shape[2:]) != (2, 3):
        raise L.AffnetB200Error("%s: %s must be [S,cap,2,3]" % (fn, name))


def _pair_args(fn, lafs1, tent, ntent, lafs2, pairs):
    """Validated (lafs1, lafs2, tent, ntent, pairs, P, tcap) in the layouts of the C ABI: every shape is checked before any tensor is
    required to be on the device."""
    lafs2 = lafs1 if lafs2 is None else lafs2
    _lafs_shape(lafs1, "lafs1", fn)
    _lafs_shape(lafs2, "lafs2", fn)
    _int_shape(tent, (None, None, 2), "tent", fn, "P,tcap,2")
    P, tcap = tent.shape[:2]
    _int_shape(ntent, (P,), "ntent", fn)
    if pairs is None:
        if not (lafs1.size(0) == lafs2.size(0) == P):
            raise L.AffnetB200Error("%s: pairs=None verifies pair p = (p, p) and needs S1 == S2 == P (%d, %d, %d)"
                                    % (fn, lafs1.size(0), lafs2.size(0), P))
    else:
        _int_shape(pairs, (P, 2), "pairs", fn)
    if P >= 1 and not 1 <= tcap <= MAX_TCAP:
        raise L.AffnetB200Error("%s: tcap must be in 1..%d (got %d)" % (fn, MAX_TCAP, tcap))
    a = L.f32c(lafs1, "lafs1")
    b = a if lafs2 is lafs1 else L.f32c(lafs2, "lafs2")
    tent = L.require_cuda(tent, "tent").to(torch.int32).contiguous()
    ntent = L.require_cuda(ntent, "ntent").to(torch.int32).contiguous()
    if pairs is not None:
        pairs = L.require_cuda(pairs, "pairs").to(torch.int32).contiguous()
    return a, b, tent, ntent, pairs, P, tcap


def find_homography_pairs(lafs1, tent, ntent, lafs2=None, pairs=None, inl_th=2.0, confidence=0.99, max_iters=50000, seed=0, affine=False,
                          laf_th=None):
    """Homography RANSAC for every pair, in one launch (ag_homography_ransac): lafs1 [S1,cap1,2,3] and lafs2 [S2,cap2,2,3] (default:
    lafs1) pixel LAFs, tent [P,tcap,2] / ntent [P] of match_snn_pairs, pairs [P,2] as given to match_snn_pairs (None: pair p = (p, p)).
    Tentative t joins the centres lafs1[i, tent[p,t,0], :, 2] and lafs2[j, tent[p,t,1], :, 2].  The defaults are those of the notebook's
    ransac_validate, findHomography(src, dst, 2.0, 0.99, 50000).  Deterministic for a seed, and a pair's result does not depend on the
    other pairs.
    -> (H [P,3,3] float32 with H[2,2] = 1, inl [P,tcap] uint8, ninl [P] int32, iters [P] int32 hypotheses evaluated).  ninl[p] is -1 for a
    pair that cannot be verified (ntent -1, an index out of range); 0 with H = 0 when it has fewer than 4 tentatives or no usable sample.
    Rows at or beyond ntent[p] are unspecified.
    affine=True (ag_homography_ransac_affine) uses the whole frames: each tentative is an affine correspondence (its centres and the local
    affinity A2 A1^-1), two of them give a hypothesis where points need four, and an inlier must also have frames that agree with H:
    D = |A1^-1 J A2 - I|_F^2 <= laf_th, J the Jacobian of H^-1 at the image-2 centre (the reference's skip-centre Frobenius distance).
    laf_th defaults to AFFINE_LAF_TH (0.5); +inf tests the centres and the frames' finiteness only.  0.5 keeps >= 97 % of the true
    matches of small synthetic warps but only 76 % on graf 1->6 (91 % at 4): for wide-baseline pairs, whose frames are noisier, a larger
    laf_th keeps more true matches (graf 1->6: 36 inliers at 0.5, 43 at 1, 45 at 2).  The frames must be oriented (OriNet or
    histogram orientation): without orientation (do_ori=False) and with an in-plane rotation between the views A2 A1^-1 is wrong, and
    the 4-point call is the right one.  iters then counts 2-AC samples, and fewer than 2 tentatives give ninl 0."""
    fn = "find_homography_pairs"
    if not float(inl_th) > 0.0 or float(inl_th) == float("inf"):
        raise L.AffnetB200Error("%s: inl_th must be finite and > 0" % fn)
    if laf_th is not None and not affine:
        raise L.AffnetB200Error("%s: laf_th is the affine test's threshold and needs affine=True" % fn)
    if affine:
        laf_th = AFFINE_LAF_TH if laf_th is None else float(laf_th)
        if not laf_th > 0.0:
            raise L.AffnetB200Error("%s: laf_th must be > 0 (+inf: no frame threshold)" % fn)
    if not 0.0 < float(confidence) < 1.0:
        raise L.AffnetB200Error("%s: confidence must be in (0, 1)" % fn)
    if int(max_iters) < 1:
        raise L.AffnetB200Error("%s: max_iters must be >= 1" % fn)
    a, b, tent, ntent, pairs, P, tcap = _pair_args(fn, lafs1, tent, ntent, lafs2, pairs)
    dev = a.device
    H = torch.empty(P, 3, 3, dtype=torch.float32, device=dev)
    inl = torch.empty(P, tcap, dtype=torch.uint8, device=dev)
    ninl = torch.empty(P, dtype=torch.int32, device=dev)
    iters = torch.empty(P, dtype=torch.int32, device=dev)
    if P == 0:
        return H, inl, ninl, iters
    if affine:
        L.check(L.lib().ag_homography_ransac_affine(L.ptr(a), a.size(0), a.size(1), L.ptr(b), b.size(0), b.size(1), L.ptr(pairs), P,
                                                    L.ptr(tent), L.ptr(ntent), tcap, float(inl_th), laf_th, float(confidence), int(max_iters),
                                                    int(seed) & (2 ** 64 - 1), L.ptr(H), L.ptr(inl), L.ptr(ninl), L.ptr(iters),
                                                    L.stream_ptr()))
        return H, inl, ninl, iters
    L.check(L.lib().ag_homography_ransac(L.ptr(a), a.size(0), a.size(1), L.ptr(b), b.size(0), b.size(1), L.ptr(pairs), P, L.ptr(tent),
                                         L.ptr(ntent), tcap, float(inl_th), float(confidence), int(max_iters), int(seed) & (2 ** 64 - 1),
                                         L.ptr(H), L.ptr(inl), L.ptr(ninl), L.ptr(iters), L.stream_ptr()))
    return H, inl, ninl, iters


def find_fundamental_pairs(lafs1, tent, ntent, lafs2=None, pairs=None, inl_th=0.5, confidence=0.99, max_iters=50000, seed=0,
                           degensac=False):
    """Fundamental-matrix RANSAC for every pair, in one launch (ag_fundamental_ransac), with the inputs of find_homography_pairs.  For
    scenes with depth, where one homography explains one plane only.  A tentative is an inlier when its Sampson distance to F is at most
    inl_th px.  inl_th = 0.5 is the notebook's alternative findFundamentalMatrix(src, dst, 0.5); confidence and max_iters are those of
    its findHomography call.  Deterministic for a seed, and a pair's result does not depend on the other pairs.
    -> (F [P,3,3] float32 with unit Frobenius norm and its largest-magnitude entry positive, inl [P,tcap] uint8, ninl [P] int32, iters [P]
    int32 7-point samples evaluated).  ninl[p] is -1 for a pair that cannot be verified (ntent -1, an index out of range); 0 with F = 0
    when it has fewer than 7 tentatives or no usable sample.  Rows at or beyond ntent[p] are unspecified.
    degensac=True (ag_fundamental_degensac) adds DEGENSAC's degeneracy test, plane-and-parallax and local optimisation, for scenes where
    one plane (a facade, a floor) carries most matches: pydegensac.findFundamentalMatrix's algorithm family, with the same inputs and
    outputs."""
    fn = "find_fundamental_pairs"
    if not float(inl_th) > 0.0 or float(inl_th) == float("inf"):
        raise L.AffnetB200Error("%s: inl_th must be finite and > 0" % fn)
    if not 0.0 < float(confidence) < 1.0:
        raise L.AffnetB200Error("%s: confidence must be in (0, 1)" % fn)
    if int(max_iters) < 1:
        raise L.AffnetB200Error("%s: max_iters must be >= 1" % fn)
    a, b, tent, ntent, pairs, P, tcap = _pair_args(fn, lafs1, tent, ntent, lafs2, pairs)
    dev = a.device
    F = torch.empty(P, 3, 3, dtype=torch.float32, device=dev)
    inl = torch.empty(P, tcap, dtype=torch.uint8, device=dev)
    ninl = torch.empty(P, dtype=torch.int32, device=dev)
    iters = torch.empty(P, dtype=torch.int32, device=dev)
    if P == 0:
        return F, inl, ninl, iters
    entry = L.lib().ag_fundamental_degensac if degensac else L.lib().ag_fundamental_ransac
    L.check(entry(L.ptr(a), a.size(0), a.size(1), L.ptr(b), b.size(0), b.size(1), L.ptr(pairs), P, L.ptr(tent), L.ptr(ntent), tcap,
                  float(inl_th), float(confidence), int(max_iters), int(seed) & (2 ** 64 - 1), L.ptr(F), L.ptr(inl), L.ptr(ninl),
                  L.ptr(iters), L.stream_ptr()))
    return F, inl, ninl, iters


def gt_correspondences_pairs(lafs1, tent, ntent, H1to2, lafs2=None, pairs=None, dist_threshold=6.0):
    """get_GT_correspondence_indexes for every pair, in one launch (ag_gt_correspondences_pairs), with the arguments of
    find_homography_pairs and H1to2 [P,3,3] (or one [3,3] for every pair).  As in the reference, the image-2 centres of all of a pair's
    tentatives are mapped through H1to2^-1 into image 1, and tentative t is true when ANY of them lies within dist_threshold px of its
    image-1 centre.  The reference's graffiti test uses 6 px.
    -> (true [P,tcap] int32: the true t in ascending order, ntrue [P] int32 (-1 for a pair that cannot be verified), min_dist [P,tcap],
    idx2 [P,tcap] int32: the nearest reprojected tentative).  Rows at or beyond ntrue / ntent are unspecified."""
    fn = "gt_correspondences_pairs"
    if not float(dist_threshold) >= 0.0:
        raise L.AffnetB200Error("%s: dist_threshold must be >= 0" % fn)
    P = tent.size(0) if isinstance(tent, torch.Tensor) and tent.dim() == 3 else -1
    if not isinstance(H1to2, torch.Tensor) or tuple(H1to2.shape) not in ((P, 3, 3), (3, 3)):
        raise L.AffnetB200Error("%s: H1to2 must be [P,3,3] or [3,3]" % fn)
    a, b, tent, ntent, pairs, P, tcap = _pair_args(fn, lafs1, tent, ntent, lafs2, pairs)
    H = L.f32c(H1to2, "H1to2")
    if H.dim() == 2:
        H = H.expand(P, 3, 3).contiguous()
    dev = a.device
    true = torch.empty(P, tcap, dtype=torch.int32, device=dev)
    ntrue = torch.empty(P, dtype=torch.int32, device=dev)
    mn = torch.empty(P, tcap, dtype=torch.float32, device=dev)
    idx2 = torch.empty(P, tcap, dtype=torch.int32, device=dev)
    if P == 0:
        return true, ntrue, mn, idx2
    L.check(L.lib().ag_gt_correspondences_pairs(L.ptr(a), a.size(0), a.size(1), L.ptr(b), b.size(0), b.size(1), L.ptr(pairs), P, L.ptr(tent),
                                                L.ptr(ntent), tcap, L.ptr(H), float(dist_threshold), L.ptr(mn), L.ptr(idx2), L.ptr(true),
                                                L.ptr(ntrue), L.stream_ptr()))
    return true, ntrue, mn, idx2


def get_GT_correspondence_indexes(LAFs1, LAFs2, H1to2, dist_threshold=4):
    """Drop-in for the reference's function (CUDA tensors): LAFs1 [n,2,3] and LAFs2 [n,2,3] matched row by row, H1to2 [3,3]
    -> (min_dist[mask], indexes in 1 [mask], nearest reprojected index in 2 [mask]) as in the reference.  It is
    gt_correspondences_pairs for one pair and reads the count back to the host."""
    fn = "get_GT_correspondence_indexes"
    for t, name in ((LAFs1, "LAFs1"), (LAFs2, "LAFs2")):
        if not isinstance(t, torch.Tensor) or t.dim() != 3 or tuple(t.shape[1:]) != (2, 3):
            raise L.AffnetB200Error("%s: %s must be [n,2,3]" % (fn, name))
    if LAFs1.size(0) != LAFs2.size(0):
        raise L.AffnetB200Error("%s: LAFs1 and LAFs2 must have the same number of rows (%d, %d)" % (fn, LAFs1.size(0), LAFs2.size(0)))
    n = LAFs1.size(0)
    dev = L.require_cuda(LAFs1, "LAFs1").device
    L.require_cuda(LAFs2, "LAFs2")
    if n == 0:
        e = torch.empty(0, dtype=torch.long, device=dev)
        return torch.empty(0, device=dev), e, e.clone()
    rows = torch.arange(n, dtype=torch.int32, device=dev)
    tent = torch.stack([rows, rows], 1)[None]
    ntent = torch.full((1,), n, dtype=torch.int32, device=dev)
    true, ntrue, mn, idx2 = gt_correspondences_pairs(LAFs1[None], tent, ntent, H1to2, LAFs2[None], None, dist_threshold)
    k = int(ntrue[0])
    keep = true[0, :k].long()
    return mn[0][keep], keep, idx2[0][keep].long()


# ---- affine-shape ground truth (get_GT_correspondence_indexes_Fro / _Fro_and_center, ReprojectionStuff.py:139-203) -------------------
def _frob_params(fn, dist_threshold, center_dist_th, scale_diff_coef, skip_center, do_up_is_up, inv_to_eye):
    if not float(dist_threshold) >= 0.0:
        raise L.AffnetB200Error("%s: dist_threshold must be >= 0" % fn)
    if center_dist_th is not None and not float(center_dist_th) >= 0.0:
        raise L.AffnetB200Error("%s: center_dist_th must be >= 0 (or None: no centre and scale gate)" % fn)
    if float(scale_diff_coef) != float(scale_diff_coef):
        raise L.AffnetB200Error("%s: scale_diff_coef must not be NaN" % fn)
    gate = center_dist_th is not None
    return L.FrobeniusParams(float(dist_threshold), float(center_dist_th) if gate else 0.0, float(scale_diff_coef), int(gate),
                             int(bool(skip_center)), int(bool(do_up_is_up)), int(bool(inv_to_eye)))


def _h_shape(fn, H1to2, P):
    if not isinstance(H1to2, torch.Tensor) or tuple(H1to2.shape) not in ((P, 3, 3), (3, 3)):
        raise L.AffnetB200Error("%s: H1to2 must be [P,3,3] or [3,3]" % fn)


def _homographies(fn, H1to2, P):
    _h_shape(fn, H1to2, P)
    H = L.f32c(H1to2, "H1to2")
    return H.expand(P, 3, 3).contiguous() if H.dim() == 2 else H


def frobenius_gt_pairs(lafs1, tent, ntent, H1to2, lafs2=None, pairs=None, dist_threshold=4.0, center_dist_th=None, scale_diff_coef=0.3,
                       skip_center=False, do_up_is_up=False, inv_to_eye=True):
    """The reference's affine-shape ground truth for every pair's tentatives, in one capturable call (ag_gt_frobenius_pairs), with the
    inputs of gt_correspondences_pairs.  Row t is lafs1[i, tent[p,t,0]]; it is compared with the frames lafs2[j, tent[p,u,1]] of all the
    pair's tentatives, mapped into image 1 through H1to2^-1 (linearised at each centre), by D = |A1^-1 A2' - I|_F^2 + |A1^-1 (t2' - t1)|^2
    (get_GT_correspondence_indexes_Fro; the 2x2 term only with skip_center).  center_dist_th (not None) selects
    get_GT_correspondence_indexes_Fro_and_center: + 1000 when the centres are >= center_dist_th px apart, + 1000 when the scale ratio
    differs from 1 by more than scale_diff_coef (no scale gate when it is <= 0), with its do_up_is_up and inv_to_eye options.  Per row
    the minimum over u (lowest index on ties, NaN ignored); true when <= dist_threshold.  A singular or non-finite side-1 frame is never
    true (min_dist +inf, idx2 0).
    -> (true [P,tcap] int32 ascending, ntrue [P] int32 (-1 for a pair that cannot be checked), min_dist [P,tcap], idx2 [P,tcap] int32).
    Rows at or beyond ntrue / ntent are unspecified."""
    fn = "frobenius_gt_pairs"
    prm = _frob_params(fn, dist_threshold, center_dist_th, scale_diff_coef, skip_center, do_up_is_up, inv_to_eye)
    _h_shape(fn, H1to2, tent.size(0) if isinstance(tent, torch.Tensor) and tent.dim() == 3 else -1)
    a, b, tent, ntent, pairs, P, tcap = _pair_args(fn, lafs1, tent, ntent, lafs2, pairs)
    H = _homographies(fn, H1to2, P)
    dev = a.device
    true = torch.empty(P, tcap, dtype=torch.int32, device=dev)
    ntrue = torch.empty(P, dtype=torch.int32, device=dev)
    mn = torch.empty(P, tcap, dtype=torch.float32, device=dev)
    idx2 = torch.empty(P, tcap, dtype=torch.int32, device=dev)
    if P == 0:
        return true, ntrue, mn, idx2
    L.check(L.lib().ag_gt_frobenius_pairs(L.ptr(a), a.size(0), a.size(1), L.ptr(b), b.size(0), b.size(1), L.ptr(pairs), P, L.ptr(tent),
                                          L.ptr(ntent), tcap, L.ptr(H), prm, L.ptr(mn), L.ptr(idx2), L.ptr(true), L.ptr(ntrue),
                                          L.stream_ptr()))
    return true, ntrue, mn, idx2


def frobenius_gt_sets(lafs1, count1, H1to2, lafs2=None, count2=None, pairs=None, dist_threshold=4.0, center_dist_th=None,
                      scale_diff_coef=0.3, skip_center=False, do_up_is_up=False, inv_to_eye=True):
    """frobenius_gt_pairs on whole detection sets (ag_gt_frobenius_sets): affine-region repeatability.  lafs1 [S1,cap1,2,3] with count1
    [S1] (DetectDescribePipeline.run's LAFs and count), lafs2 [S2,cap2,2,3] with count2 [S2] (default: lafs1, count1), pairs [P,2]
    (None: pair p = (p, p)), H1to2 [P,3,3] or [3,3].  Pair p = (i, j) checks rows 0..count1[i]-1 of set i against rows 0..count2[j]-1
    of set j; the counts are read on the device.
    -> (true [P,cap1] int32 ascending, ntrue [P] int32 (-1 when i or j is out of range or a count lies outside 0..cap), min_dist
    [P,cap1], idx2 [P,cap1] int32: the nearest row of set j).  Rows at or beyond ntrue / count1[i] are unspecified."""
    fn = "frobenius_gt_sets"
    prm = _frob_params(fn, dist_threshold, center_dist_th, scale_diff_coef, skip_center, do_up_is_up, inv_to_eye)
    if lafs2 is None:
        lafs2, count2 = lafs1, count1 if count2 is None else count2
    elif count2 is None:
        raise L.AffnetB200Error("%s: count2 is required with lafs2" % fn)
    _lafs_shape(lafs1, "lafs1", fn)
    _lafs_shape(lafs2, "lafs2", fn)
    S1, cap1, S2, cap2 = lafs1.size(0), lafs1.size(1), lafs2.size(0), lafs2.size(1)
    _int_shape(count1, (S1,), "count1", fn)
    _int_shape(count2, (S2,), "count2", fn)
    if pairs is None:
        if S1 != S2:
            raise L.AffnetB200Error("%s: pairs=None checks pair p = (p, p) and needs S1 == S2 (%d, %d)" % (fn, S1, S2))
        P = S1
    else:
        _int_shape(pairs, (None, 2), "pairs", fn, "P,2")
        P = pairs.size(0)
    if P >= 1 and not (1 <= cap1 <= MAX_TCAP and cap2 >= 1):
        raise L.AffnetB200Error("%s: cap1 must be in 1..%d and cap2 >= 1 (got %d, %d)" % (fn, MAX_TCAP, cap1, cap2))
    H = _homographies(fn, H1to2, P)
    a = L.f32c(lafs1, "lafs1")
    b = a if lafs2 is lafs1 else L.f32c(lafs2, "lafs2")
    c1 = L.require_cuda(count1, "count1").to(torch.int32).contiguous()
    c2 = c1 if count2 is count1 else L.require_cuda(count2, "count2").to(torch.int32).contiguous()
    if pairs is not None:
        pairs = L.require_cuda(pairs, "pairs").to(torch.int32).contiguous()
    dev = a.device
    true = torch.empty(P, cap1, dtype=torch.int32, device=dev)
    ntrue = torch.empty(P, dtype=torch.int32, device=dev)
    mn = torch.empty(P, cap1, dtype=torch.float32, device=dev)
    idx2 = torch.empty(P, cap1, dtype=torch.int32, device=dev)
    if P == 0:
        return true, ntrue, mn, idx2
    L.check(L.lib().ag_gt_frobenius_sets(L.ptr(a), S1, cap1, L.ptr(c1), L.ptr(b), S2, cap2, L.ptr(c2), L.ptr(pairs), P, L.ptr(H), prm,
                                         L.ptr(mn), L.ptr(idx2), L.ptr(true), L.ptr(ntrue), L.stream_ptr()))
    return true, ntrue, mn, idx2


def _reproject(lafs, H, invert, up_is_up):
    """ag_reproject_lafs of one set lafs [n,2,3] (n >= 1) through H [3,3] (its inverse with invert) -> [n,2,3]."""
    a = L.f32c(lafs, "LAFs")
    Hc = L.f32c(H, "H1to2")
    out = torch.empty_like(a)
    L.check(L.lib().ag_reproject_lafs(L.ptr(a), 1, a.size(0), L.ptr(Hc), int(invert), int(up_is_up), L.ptr(out), L.stream_ptr()))
    return out


def _laf_rows(fn, t, name):
    if not isinstance(t, torch.Tensor) or t.dim() != 3 or tuple(t.shape[1:]) != (2, 3):
        raise L.AffnetB200Error("%s: %s must be [n,2,3]" % (fn, name))


def _square_h(fn, H1to2):
    if not isinstance(H1to2, torch.Tensor) or tuple(H1to2.shape) != (3, 3):
        raise L.AffnetB200Error("%s: H1to2 must be [3,3]" % fn)


def reprojectLAFs(LAFs1, H1to2, return_LHFs=False):
    """Drop-in for the reference's function (CUDA tensors): LAFs1 [n,2,3] mapped through H1to2 [3,3], the 2x2 part by linH at each
    centre -> [n,2,3], or [n,3,3] with the row [0, 0, 1] when return_LHFs.  In fp64, each value rounded once to fp32."""
    fn = "reprojectLAFs"
    _laf_rows(fn, LAFs1, "LAFs1")
    _square_h(fn, H1to2)
    L.require_cuda(LAFs1, "LAFs1")
    out = _reproject(LAFs1, H1to2, False, False) if LAFs1.size(0) else torch.empty(0, 2, 3, device=LAFs1.device)
    if return_LHFs:
        last = torch.tensor([0.0, 0.0, 1.0], device=out.device).expand(out.size(0), 1, 3)
        out = torch.cat([out, last], dim=1)
    return out


def _frob_dropin(fn, LAFs1, LAFs2, H1to2, dist_threshold, center_dist_th, scale_diff_coef, skip_center, do_up_is_up, inv_to_eye):
    _laf_rows(fn, LAFs1, "LAFs1")
    _laf_rows(fn, LAFs2, "LAFs2")
    _square_h(fn, H1to2)
    _frob_params(fn, dist_threshold, center_dist_th, scale_diff_coef, skip_center, do_up_is_up, inv_to_eye)
    dev = L.require_cuda(LAFs1, "LAFs1").device
    L.require_cuda(LAFs2, "LAFs2")
    n1, n2 = LAFs1.size(0), LAFs2.size(0)
    if n1 == 0 or n2 == 0:
        e = torch.empty(0, dtype=torch.long, device=dev)
        return torch.empty(0, device=dev), e, e.clone()
    c1 = torch.full((1,), n1, dtype=torch.int32, device=dev)
    c2 = torch.full((1,), n2, dtype=torch.int32, device=dev)
    true, ntrue, mn, idx2 = frobenius_gt_sets(LAFs1[None], c1, H1to2, LAFs2[None], c2, None, dist_threshold, center_dist_th,
                                              scale_diff_coef, skip_center, do_up_is_up, inv_to_eye)
    keep = true[0, :int(ntrue[0])].long()
    return mn[0][keep], keep, idx2[0][keep].long()


def get_GT_correspondence_indexes_Fro(LAFs1, LAFs2, H1to2, dist_threshold=4, skip_center_in_Fro=False):
    """Drop-in for the reference's function (CUDA tensors): every LAFs1 [n1,2,3] row against all LAFs2 [n2,2,3] rows mapped into
    image 1 through H1to2^-1 -> (min_dist[mask], indexes in 1 [mask], nearest index in 2 [mask]).  It is frobenius_gt_sets for one pair
    and reads the count back to the host.  It returns the intended distance matrix's minima where the reference scrambles its rows, and a
    singular row of LAFs1 is never true where the reference raises (DESIGN.md, Frobenius quirks)."""
    return _frob_dropin("get_GT_correspondence_indexes_Fro", LAFs1, LAFs2, H1to2, dist_threshold, None, 0.0, skip_center_in_Fro, False,
                        True)


def get_GT_correspondence_indexes_Fro_and_center(LAFs1, LAFs2, H1to2, dist_threshold=4, center_dist_th=2.0, scale_diff_coef=0.3,
                                                 skip_center_in_Fro=False, do_up_is_up=False, return_LAF2_in_1=False, inv_to_eye=True):
    """Drop-in for the reference's function (CUDA tensors), as get_GT_correspondence_indexes_Fro with its centre and scale gates;
    scale_diff_coef <= 0 means no scale gate (the reference raises).  With return_LAF2_in_1 a fourth output, LAFs2 mapped into image 1
    [n2,2,3] (rectified with do_up_is_up), as ag_reproject_lafs computes it."""
    fn = "get_GT_correspondence_indexes_Fro_and_center"
    if center_dist_th is None:
        raise L.AffnetB200Error("%s: center_dist_th must be a number" % fn)
    out = _frob_dropin(fn, LAFs1, LAFs2, H1to2, dist_threshold, center_dist_th, scale_diff_coef, skip_center_in_Fro, do_up_is_up,
                       inv_to_eye)
    if return_LAF2_in_1:
        l2 = _reproject(LAFs2, H1to2, True, do_up_is_up) if LAFs2.size(0) else torch.empty(0, 2, 3, device=LAFs2.device)
        out = out + (l2,)
    return out
