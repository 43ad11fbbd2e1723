"""ReprojectionStuff.py counterpart for verifying matches on the device: the reference's ground-truth check
(get_GT_correspondence_indexes, ReprojectionStuff.py:126-137), homography RANSAC (the notebook's ransac_validate) and
fundamental-matrix RANSAC (its findFundamentalMatrix alternative, also as DEGENSAC), for one pair or for every pair of a batch in one call.  The batched calls take DetectDescribePipeline.run's LAFs and
Losses.match_snn_pairs' (tent, ntent) as they are, never synchronise with the host, and are capturable in the same CUDA graph."""
import torch

from . import _lib as L

MAX_TCAP = 4194240   # ag_match_pairs' cap1 limit


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


def find_homography_pairs(lafs1, tent, ntent, lafs2=None, pairs=None, inl_th=2.0, confidence=0.99, max_iters=50000, seed=0):
    """Homography RANSAC for every pair, in one launch (ag_homography_ransac): lafs1 [S1,cap1,2,3] and lafs2 [S2,cap2,2,3] (default:
    lafs1) pixel LAFs, tent [P,tcap,2] / ntent [P] of match_snn_pairs, pairs [P,2] as given to match_snn_pairs (None: pair p = (p, p)).
    Tentative t joins the centres lafs1[i, tent[p,t,0], :, 2] and lafs2[j, tent[p,t,1], :, 2].  The defaults are those of the notebook's
    ransac_validate, findHomography(src, dst, 2.0, 0.99, 50000).  Deterministic for a seed, and a pair's result does not depend on the
    other pairs.
    -> (H [P,3,3] float32 with H[2,2] = 1, inl [P,tcap] uint8, ninl [P] int32, iters [P] int32 hypotheses evaluated).  ninl[p] is -1 for a
    pair that cannot be verified (ntent -1, an index out of range); 0 with H = 0 when it has fewer than 4 tentatives or no usable sample.
    Rows at or beyond ntent[p] are unspecified."""
    fn = "find_homography_pairs"
    if not float(inl_th) > 0.0 or float(inl_th) == float("inf"):
        raise L.AffnetB200Error("%s: inl_th must be finite and > 0" % fn)
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
