"""CPU tests (-m "not gpu") of the Frobenius ground truth (ag_gt_frobenius_pairs / _sets): the restatement (tests/frobenius_restated.py)
against the reference's outputs in tests/golden/frobenius.npz, the reference's quirks that the device does not copy, and the refusals
before any CUDA call."""
import numpy as np
import pytest
import torch

import frobenius_restated as FR
from helpers import gold

CASES = {"fro": {}, "fro_skip": dict(skip_center=True), "fc": dict(center_dist_th=2.0), "fc_skip": dict(center_dist_th=2.0, skip_center=True),
         "fc_up": dict(center_dist_th=2.0, do_up_is_up=True), "fc_noinv": dict(center_dist_th=2.0, inv_to_eye=False),
         "fc_noinv_skip": dict(center_dist_th=2.0, inv_to_eye=False, skip_center=True)}
# Rows whose result differs from the reference's by a decision within rounding of its threshold.  Row 175 of graf img1 has its
# nearest frame 1.992 px away: the expanded centre distance, whose cancellation error at |t| ~ 370 px is about 0.03 px in fp32, puts it
# at or beyond center_dist_th = 2 in the reference and below it here.  Row 2006 with inv_to_eye = False has two columns whose expanded
# distances lie within their bound of each other: a near tie.
EXEMPT = {("set", k): {175} for k in ("fc", "fc_skip", "fc_up", "fc_noinv_skip")}
EXEMPT[("set", "fc_noinv")] = {175, 2006}
TH = 4.0   # the reference's default dist_threshold


def graf_case(mode):
    z, m = gold("frobenius.npz"), gold("graf_match.npz")
    if mode == "set":
        return z["lafs1"], z["lafs6"], z["H1to6"]
    return z["lafs1"][m["noori_t1"]], z["lafs6"][m["noori_t2"]], z["H1to6"]


def gate_uncertain(r, c, i, j, prm):
    """The gate of (i, j) could round either way: the centre distance within the expanded form's bound (8 u (|t| + |t'|)^2 on the
    square) of center_dist_th, or |1 - s'/s| within 8 u of scale_diff_coef."""
    if not prm.gate:
        return False
    cd = float(FR.centre_dist({k: v[i:i + 1] for k, v in r.items()}, {k: v[j:j + 1] for k, v in c.items()})[0, 0])
    mag = (abs(float(r["x"][i])) + abs(float(r["y"][i])) + abs(float(c["x"][j])) + abs(float(c["y"][j]))) ** 2
    ratio = abs(1.0 - float(c["s"][j]) / float(r["s1e"][i]))
    return abs(cd * cd - float(prm.cth) ** 2) <= 8 * FR.U32 * mag or abs(ratio - float(prm.coef)) <= 8 * FR.U32 * max(1.0, ratio)


def agreement(l1, l2, H, kw, ref_min, ref_i1, ref_i2):
    """-> the rows that differ from the reference (min_dist beyond the bound, idx2, or the decision at TH), after asserting that each
    is a near tie, near TH, or a gate within rounding; and the rows the reference leaves out (a NaN in the row)."""
    prm = FR.Params(dist_threshold=np.inf, **kw)
    r, c = FR.rows(l1, prm), FR.cols(l2, H, prm)
    D = FR.distances(r, c, prm)
    mn, idx, _ = FR.reduce_rows(D, np.inf)
    Du = FR.distances(r, c, prm, gated=False)
    B = FR.d_bound(Du, r, c, prm) if prm.inv else FR.d_bound_expanded(Du, r, c)
    missing = sorted(set(range(len(l1))) - set(ref_i1.tolist()))
    assert all(np.isnan(D[i]).any() or not np.isfinite(mn[i]) for i in missing)
    differ = set()
    for k, i in enumerate(ref_i1.tolist()):
        j, rj = int(idx[i]), int(ref_i2[k])
        b = max(B[i, j], B[i, rj])
        same_val = abs(float(mn[i]) - float(ref_min[k])) <= b
        if same_val and j == rj and (mn[i] <= TH) == (ref_min[k] <= TH):
            continue
        differ.add(i)
        near_tie = abs(float(D[i, rj]) - float(mn[i])) <= B[i, j] + B[i, rj]
        near_th = abs(float(ref_min[k]) - TH) <= b
        assert (same_val and (near_tie or near_th)) or gate_uncertain(r, c, i, j, prm) or gate_uncertain(r, c, i, rj, prm), (i, j, rj)
    return differ, missing


@pytest.mark.parametrize("mode", ["set", "tent"])
@pytest.mark.parametrize("case", list(CASES))
def test_restatement_agrees_with_the_reference(mode, case):
    z = gold("frobenius.npz")
    l1, l2, H = graf_case(mode)
    differ, missing = agreement(l1, l2, H, CASES[case], z["%s_%s_min" % (mode, case)], z["%s_%s_i1" % (mode, case)], z["%s_%s_i2" % (mode, case)])
    assert differ == EXEMPT.get((mode, case), set())
    assert missing == []


@pytest.mark.parametrize("mode", ["set", "tent"])
def test_reprojection_agrees_with_the_reference(mode):
    z = gold("frobenius.npz")
    _, l2, H = graf_case(mode)
    ours = FR.reproject_lafs(l2, H, True, False)
    ref = z["%s_l2in1" % mode]
    # the reference maps in fp32 through an fp32 H^-1 (cond(H1to6) ~ 4.5e5): centres within 1e-2 px, 2x2 parts within 1e-5 relative
    assert np.abs(ours[:, :, 2] - ref[:, :, 2]).max() < 1e-2
    assert (np.abs(ours[:, :, :2] - ref[:, :, :2]) <= 1e-5 * np.abs(ref[:, :, :2]).max(axis=(1, 2), keepdims=True)).all()


def test_nan_and_infinite_columns_never_win():
    """The random case: side-2 frame 2 has a NaN entry and frame 5 an infinite centre.  Its matrix equals the reference's within the
    bound wherever the reference's is a number; the reference's torch.min returns NaN for every row (so it keeps none), the device
    ignores NaN."""
    z = gold("frobenius.npz")
    prm = FR.Params(dist_threshold=np.inf)
    r, c = FR.rows(z["rnd_l1"], prm), FR.cols(z["rnd_l2"], z["rnd_H"], prm)
    D = FR.distances(r, c, prm)
    ref = z["rnd_D1"]
    assert np.array_equal(np.isnan(D), np.isnan(ref)) and np.isnan(D[:, 2]).all()
    ok = np.isfinite(ref)
    assert (np.abs(D[ok] - ref[ok]) <= FR.d_bound(D, r, c, prm)[ok]).all()
    assert len(z["rnd_fro_i1"]) == 0 and len(z["rnd_fc_i1"]) == 0
    mn, idx, _ = FR.reduce_rows(D, np.inf)
    assert np.isfinite(mn).all() and not np.isin(idx, [2, 5]).any()


@pytest.mark.parametrize("case", ["tent", "rnd"])
def test_batch_size_2_scrambles_the_reference_matrix(case):
    """Quirk 1: with batch_size = 2 the reference returns out[s + a, b] = D[s + f % 2, f // 2], f = a len2 + b, for each full batch
    starting at row s (the last, odd row is D's)."""
    z = gold("frobenius.npz")
    D1, D2 = z[case + "_D1"], z[case + "_D2"]
    n1, n2 = D1.shape
    want = D1.copy()
    for s in range(0, n1 - 1, 2):
        f = np.arange(2 * n2).reshape(2, n2)
        want[s:s + 2] = D1[s + f % 2, f // 2]
    assert np.array_equal(want, D2, equal_nan=True) and not np.array_equal(D1, D2, equal_nan=True)


def test_scale_diff_coef_zero_and_singular_rows():
    """Quirks 2 and 3: the reference raises for scale_diff_coef = 0 and for a singular row of LAFs1.  Here scale_diff_coef <= 0 means no
    scale gate, and a singular row is never true."""
    z = gold("frobenius.npz")
    assert str(z["err_scale0"]) == "UnboundLocalError" and "LinAlgError" in str(z["err_singular"])
    l1, l2, H = z["rnd_l1"], z["rnd_l2"], z["rnd_H"]
    off = FR.frobenius(l1, l2, H, FR.Params(np.inf, 2.0, 0.0))
    for coef in (-1.0, 1e30):
        other = FR.frobenius(l1, l2, H, FR.Params(np.inf, 2.0, coef))
        assert all(np.array_equal(a, b) for a, b in zip(off, other))
    sing = np.concatenate([l1[:3], np.array([[[1.0, 2.0, 5.0], [2.0, 4.0, 5.0]]], np.float32)])
    mn, idx, true = FR.frobenius(sing, l2, H, FR.Params(4.0))
    assert mn[3] == np.inf and idx[3] == 0 and 3 not in true.tolist() and np.isfinite(mn[:3]).all()


def test_refusals_before_any_cuda_call():
    from affnet_b200 import _lib as L
    from affnet_b200.ReprojectionStuff import (frobenius_gt_pairs, frobenius_gt_sets, get_GT_correspondence_indexes_Fro,
                                               get_GT_correspondence_indexes_Fro_and_center, reprojectLAFs)
    lafs = torch.zeros(2, 5, 2, 3)
    tent = torch.zeros(2, 4, 2, dtype=torch.int32)
    nt = torch.zeros(2, dtype=torch.int32)
    cnt = torch.zeros(2, dtype=torch.int32)
    H = torch.eye(3)
    nan = float("nan")
    for fn, kw, msg in [
        (frobenius_gt_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, H1to2=H, dist_threshold=nan), "dist_threshold"),
        (frobenius_gt_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, H1to2=H, dist_threshold=-1.0), "dist_threshold"),
        (frobenius_gt_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, H1to2=H, center_dist_th=nan), "center_dist_th"),
        (frobenius_gt_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, H1to2=H, center_dist_th=-2.0), "center_dist_th"),
        (frobenius_gt_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, H1to2=H, scale_diff_coef=nan), "scale_diff_coef"),
        (frobenius_gt_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, H1to2=torch.eye(3)[None]), r"H1to2 must be \[P,3,3\] or \[3,3\]"),
        (frobenius_gt_pairs, dict(lafs1=lafs[:, :, :1], tent=tent, ntent=nt, H1to2=H), r"lafs1 must be \[S,cap,2,3\]"),
        (frobenius_gt_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, H1to2=H), "must be a CUDA tensor"),
        (frobenius_gt_sets, dict(lafs1=lafs, count1=cnt, H1to2=H, dist_threshold=nan), "dist_threshold"),
        (frobenius_gt_sets, dict(lafs1=lafs, count1=cnt[:1], H1to2=H), r"count1 must be an integer tensor \[2\]"),
        (frobenius_gt_sets, dict(lafs1=lafs, count1=cnt.float(), H1to2=H), "count1 must be an integer tensor"),
        (frobenius_gt_sets, dict(lafs1=lafs, count1=cnt, H1to2=H, lafs2=lafs), "count2 is required"),
        (frobenius_gt_sets, dict(lafs1=lafs, count1=cnt, H1to2=H, lafs2=lafs[:1], count2=cnt[:1]), "needs S1 == S2"),
        (frobenius_gt_sets, dict(lafs1=lafs, count1=cnt, H1to2=torch.eye(3).expand(3, 3, 3)), r"H1to2 must be \[P,3,3\]"),
        (frobenius_gt_sets, dict(lafs1=lafs, count1=cnt, H1to2=H), "must be a CUDA tensor"),
        (get_GT_correspondence_indexes_Fro, dict(LAFs1=lafs[0], LAFs2=lafs[0], H1to2=H), "must be a CUDA tensor"),
        (get_GT_correspondence_indexes_Fro, dict(LAFs1=lafs, LAFs2=lafs[0], H1to2=H), r"LAFs1 must be \[n,2,3\]"),
        (get_GT_correspondence_indexes_Fro_and_center, dict(LAFs1=lafs[0], LAFs2=lafs[0], H1to2=H, center_dist_th=None), "center_dist_th"),
        (reprojectLAFs, dict(LAFs1=lafs[0], H1to2=H[None]), r"H1to2 must be \[3,3\]"),
    ]:
        with pytest.raises(L.AffnetB200Error, match=msg):
            fn(**kw)
