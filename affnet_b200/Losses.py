"""Losses.py counterpart on the evaluation side of the hot path: distance_matrix_vector (Losses.py:5-13) and the
second-nearest-neighbour ratio matcher of train_AffNet_test_on_graffity.py:292-298."""
import torch

from . import _lib as L


def distance_matrix_vector(anchor, positive):
    """[n1,D], [n2,D] CUDA float32 -> [n1,n2] sqrt(|a|^2 + |b|^2 - 2 a.b + 1e-6)."""
    a, b = L.f32c(anchor, "anchor"), L.f32c(positive, "positive")
    out = torch.empty(a.size(0), b.size(0), dtype=torch.float32, device=a.device)
    if a.size(0) and b.size(0):
        L.check(L.lib().ag_distance_matrix(L.ptr(a), a.size(0), L.ptr(b), b.size(0), a.size(1), L.ptr(out), L.stream_ptr()))
    return out


def match_snn(descriptors1, descriptors2, SNN_threshold=0.8):
    """-> (tent_matches_in_1, tent_matches_in_2, min_dist, min_2nd_dist) exactly as the reference's test() computes them,
    including `dist_matrix[:, idxs_in_2] = 100000` before the second minimum."""
    a, b = L.f32c(descriptors1, "descriptors1"), L.f32c(descriptors2, "descriptors2")
    n1, n2 = a.size(0), b.size(0)
    dev = a.device
    if a.dim() != 2 or b.dim() != 2 or (n1 and n2 and a.size(1) != b.size(1)):
        raise L.AffnetB200Error("match_snn: descriptors must be [n1,D] and [n2,D] with the same D")
    if n1 == 0 or n2 == 0:     # the reference returns empty matches
        e = torch.empty(0, dtype=torch.long, device=dev)
        return e, e.clone(), torch.empty(n1, device=dev), torch.empty(n1, device=dev)
    nb = L.lib().ag_match_snn_workspace_bytes(n1, n2)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    idx = torch.empty(n1, dtype=torch.int32, device=dev)
    mn = torch.empty(n1, dtype=torch.float32, device=dev)
    sec = torch.empty(n1, dtype=torch.float32, device=dev)
    keep = torch.empty(n1, dtype=torch.uint8, device=dev)
    L.check(L.lib().ag_match_snn(L.ptr(a), n1, L.ptr(b), n2, a.size(1), float(SNN_threshold), L.ptr(ws), nb, L.ptr(idx), L.ptr(mn), L.ptr(sec),
                                 L.ptr(keep), L.stream_ptr()))
    mask = keep.bool()
    return torch.arange(n1, device=dev)[mask], idx.long()[mask], mn, sec


def _counts(c, S, name):
    if c is None:
        return None
    if not isinstance(c, torch.Tensor) or c.shape != (S,) or c.dtype.is_floating_point or c.dtype.is_complex or c.dtype == torch.bool:
        raise L.AffnetB200Error("match_snn_pairs: %s must be an integer tensor [%d]" % (name, S))
    return L.require_cuda(c, name).to(torch.int32).contiguous()


def match_snn_pairs(desc1, count1=None, desc2=None, count2=None, pairs=None, SNN_threshold=0.8):
    """match_snn for a list of image pairs in one device call, without a host synchronisation (capturable in a CUDA graph together with
    DetectDescribePipeline.run).  desc1 [S1,cap1,D] with count1 [S1] (None: every image has cap1 rows), desc2 [S2,cap2,D] with count2
    [S2] (default: set 1), pairs [P,2] CUDA integer tensor of (image of set 1, image of set 2) (None: pair p = (p, p)).  Takes the
    pipeline's (desc, count) and DescriptorExchange.last()'s (desc, count) as they are.
    -> (tent [P,cap1,2] int32, ntent [P] int32, min_dist [P,cap1], min_2nd_dist [P,cap1]): tent[p, :ntent[p]] = (row, nearest column) of
    the kept rows in ascending row order, the batched form of match_snn's (tent_matches_in_1, tent_matches_in_2).  ntent[p] is -1 for a
    pair with an index out of range or a count of -1 (candidate overflow), 0 when either image has no rows.  Rows beyond the counts are
    unspecified."""
    if desc2 is None:
        desc2, count2 = desc1, count1 if count2 is None else count2
    for d, name in ((desc1, "desc1"), (desc2, "desc2")):
        if not isinstance(d, torch.Tensor) or d.dim() != 3:
            raise L.AffnetB200Error("match_snn_pairs: %s must be [S,cap,D]" % name)
    if desc1.size(2) != desc2.size(2):
        raise L.AffnetB200Error("match_snn_pairs: desc1 and desc2 have different D (%d, %d)" % (desc1.size(2), desc2.size(2)))
    S1, cap1, D = desc1.shape
    S2, cap2 = desc2.shape[:2]
    c1, c2 = _counts(count1, S1, "count1"), _counts(count2, S2, "count2")
    if pairs is None:
        if S1 != S2:
            raise L.AffnetB200Error("match_snn_pairs: pairs=None matches image p with image p and needs S1 == S2 (%d, %d)" % (S1, S2))
        P = S1
    else:
        if (not isinstance(pairs, torch.Tensor) or pairs.dim() != 2 or pairs.size(1) != 2 or pairs.dtype.is_floating_point
                or pairs.dtype.is_complex or pairs.dtype == torch.bool):
            raise L.AffnetB200Error("match_snn_pairs: pairs must be an integer tensor [P,2]")
        pairs = L.require_cuda(pairs, "pairs").to(torch.int32).contiguous()
        P = pairs.size(0)
    a = L.f32c(desc1, "desc1")
    b = a if desc2 is desc1 else L.f32c(desc2, "desc2")
    dev = a.device
    tent = torch.empty(P, cap1, 2, dtype=torch.int32, device=dev)
    ntent = torch.empty(P, dtype=torch.int32, device=dev)
    mn = torch.empty(P, cap1, dtype=torch.float32, device=dev)
    sec = torch.empty(P, cap1, dtype=torch.float32, device=dev)
    if P == 0:
        return tent, ntent, mn, sec
    idx = torch.empty(P, cap1, dtype=torch.int32, device=dev)
    keep = torch.empty(P, cap1, dtype=torch.uint8, device=dev)
    nb = L.lib().ag_match_pairs_workspace_bytes(S1, cap1, S2, cap2, P)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    L.check(L.lib().ag_match_pairs(L.ptr(a), L.ptr(c1), S1, cap1, L.ptr(b), L.ptr(c2), S2, cap2, D, L.ptr(pairs), P, float(SNN_threshold),
                                   L.ptr(ws), nb, L.ptr(idx), L.ptr(mn), L.ptr(sec), L.ptr(keep), L.ptr(tent), L.ptr(ntent), L.stream_ptr()))
    return tent, ntent, mn, sec
