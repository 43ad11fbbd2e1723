"""GPU tests (-m gpu) of the given-keypoints mode: ag_pipeline_create_given / ag_pipeline_run_given (DescribeGivenPipeline) and
ag_ells_to_lafs (LAF.ells2LAFsT).  The pipeline is pinned bit for bit to its own steps called through the existing entry points, to the
detect pipeline's descriptors when fed its own keypoints, and to the oracle's composition (tests/given_restated.py) within the end-to-end
tolerances; outputs start as sentinels, and rows at or beyond a count must keep them."""
import ctypes as C

import numpy as np
import pytest
import torch

import given_restated as G
from helpers import SENTINEL, TOL, gold, gray_from_rgb, load_weights

pytestmark = pytest.mark.gpu

DEV = "cuda"
ISENT = int(SENTINEL)
W = load_weights()


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


@pytest.fixture(scope="module")
def nets():
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    return a.eval().to(DEV), o.eval().to(DEV), h.eval().to(DEV)


def crop_img():
    return gray_from_rgb(gold("graf_crop.npz")["rgb"])


def graf_1024():
    import cv2
    return gray_from_rgb(cv2.resize(gold("graf_full.npz")["rgb"], (1024, 768), interpolation=cv2.INTER_LINEAR))


def upright(xs, ys, ss):
    out = torch.zeros(len(xs), 2, 3)
    out[:, 0, 0] = torch.as_tensor(ss, dtype=torch.float32)
    out[:, 1, 1] = out[:, 0, 0]
    out[:, 0, 2] = torch.as_tensor(xs, dtype=torch.float32)
    out[:, 1, 2] = torch.as_tensor(ys, dtype=torch.float32)
    return out


def random_keypoints(n, H, W_, seed, border=True):
    """Upright keypoints spread over the image, the last ones near, on and across the border (and outside the image)."""
    g = torch.Generator().manual_seed(seed)
    s = torch.exp(torch.rand(n, generator=g) * 2.5) * 3.0
    x = torch.rand(n, generator=g) * W_
    y = torch.rand(n, generator=g) * H
    if border:
        k = n // 8
        x[:k] = torch.tensor([-5.0, 0.0, 1.0, 3.0, W_ - 1.0, W_ + 0.0, W_ + 4.0, 10.0] * (k // 8 + 1))[:k]
        s[:k] = torch.tensor([2.0, 3.0, 1.0, 3.0, 4.0, 2.0, 6.0, 10.0] * (k // 8 + 1))[:k]
    return upright(x, y, s)


def hand_crafted(kind):
    from affnet_b200.HandCraftedModules import AffineShapeEstimator, OrientationDetector
    return AffineShapeEstimator(patch_size=19) if kind == "shape" else OrientationDetector(patch_size=19)


def modules(nets, shape, ori, desc):
    from affnet_b200.pytorch_sift import SIFTNet
    a, o, h = nets
    aff = a if shape == "affnet" else (hand_crafted("shape") if shape == "baumberg" else None)
    orin = o if ori == "orinet" else (hand_crafted("ori") if ori == "histogram" else None)
    hd = SIFTNet(patch_size=int(desc[4:])) if desc.startswith("sift") else h
    return aff, orin, hd


def given_pipe(B, H, W_, nets, shape, iters, ori, desc, C_):
    from affnet_b200.pipeline import DescribeGivenPipeline
    aff, orin, hd = modules(nets, shape, ori, desc)
    p = DescribeGivenPipeline(B, H, W_, aff, hd, orin, capacity=C_, do_ori=ori is not None, num_Baum_iters=iters if shape else 0)
    p.lafs.fill_(SENTINEL); p.desc.fill_(SENTINEL); p.src.fill_(ISENT); p.count.fill_(ISENT)
    return p


def bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ---- 1. identity: the detect pipeline's own keypoints, no estimator step -----------------------------------------------------------------
@pytest.mark.parametrize("desc", ["hardnet", "sift32"])
def test_identity_on_the_detect_pipelines_keypoints(L, nets, desc):
    """DetectDescribePipeline's (lafs, count) fed back with no shape and no orientation step: the same descriptors bit for bit, the LAFs
    unchanged and src = arange(count)."""
    from affnet_b200.pipeline import DetectDescribePipeline
    img = crop_img()
    imgs = torch.cat([img, torch.flip(img, dims=[3])], 0).to(DEV).contiguous()
    B, H, W_ = 2, img.size(2), img.size(3)
    a, o, h = nets
    hd = modules(nets, None, None, desc)[2]
    det = DetectDescribePipeline(B, H, W_, a, hd, o, num_features=300, do_ori=True)
    lafs, _, d, cnt = det.run(imgs)
    g = given_pipe(B, H, W_, nets, None, 0, None, desc, 300)
    gl, src, gd, gc = g.run(imgs, lafs, cnt)
    torch.cuda.synchronize()
    assert torch.equal(gc, cnt)
    for b in range(B):
        n = int(cnt[b])
        assert n > 100
        assert bits_equal(gd[b, :n], d[b, :n]) and bits_equal(gl[b, :n], lafs[b, :n])
        assert torch.equal(src[b, :n].cpu(), torch.arange(n, dtype=torch.int32))
        assert (gd[b, n:] == SENTINEL).all() and (src[b, n:] == ISENT).all()


# ---- 2. composition of the existing entry points, bit for bit -----------------------------------------------------------------------------
MODES = [("affnet", 1, "orinet", "hardnet"), ("affnet", 3, "histogram", "sift41"), ("affnet", 1, None, "sift41"),
         ("baumberg", 1, None, "hardnet"), ("baumberg", 16, "orinet", "sift41"), (None, 0, "histogram", "hardnet"),
         (None, 0, "orinet", "sift41"), (None, 0, None, "hardnet"), ("affnet", 3, "orinet", "hardnet")]


def composition(L, nets, plan, pyr, lafs_in, counts, C_, shape, iters, ori, desc, H, W_):
    """The given pipeline's steps through the existing entry points, on the same pyramid."""
    lib, st = L.lib(), L.stream_ptr()
    a, o, h = nets
    B = counts.numel()
    n = B * C_
    ms = float(min(H, W_))
    na, nx, ny = float(np.float32(1.0) / np.float32(ms)), float(np.float32(1.0 / W_)), float(np.float32(1.0 / H))
    ws_bytes = max(lib.ag_net_workspace_bytes(k, n) for k in (0, 1, 2))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)

    def empty(*shape_, dtype=torch.float32):
        return torch.full(shape_, SENTINEL if dtype == torch.float32 else ISENT, dtype=dtype, device=DEV)

    def level(src, ps):
        oc, lv = empty(B, C_, dtype=torch.int32), empty(B, C_, dtype=torch.int32)
        L.check(lib.ag_pyramid_level_for_lafs(plan, L.ptr(src), n, ps, L.ptr(oc), L.ptr(lv), st))
        return oc, lv

    def scale(src, ac, xc, yc):
        out = empty(B, C_, 2, 3)
        L.check(lib.ag_lafs_scale(L.ptr(src), L.ptr(out), n, ac, xc, yc, st))
        return out

    def net(mod, lafs, oc, lv, cnt, width):
        out = empty(B, C_, width)
        L.check(lib.ag_net_forward_pyr(mod.handle(), plan, L.ptr(pyr), L.ptr(lafs), L.ptr(oc), L.ptr(lv), L.ptr(cnt), C_, L.ptr(out),
                                       L.ptr(ws), ws_bytes, st))
        return out

    cnt = counts.to(DEV, torch.int32).contiguous()
    src = torch.arange(C_, dtype=torch.int32, device=DEV).repeat(B, 1)
    if shape is None and ori is None:
        dl = lafs_in
    else:
        oct1, lvl1 = level(lafs_in, 32)
        nl = scale(lafs_in, na, nx, ny)
        if shape is not None:
            if shape == "baumberg":
                gk = np.zeros((19, 19), np.float32)
                L.check(lib.ag_circular_gauss_kernel(19, (19 / 2.0) / 3.0, gk.ctypes.data_as(C.c_void_p)))
                A = empty(B, C_, 4)
                L.check(lib.ag_debug_baumberg_pyr(plan, L.ptr(pyr), L.ptr(nl), L.ptr(oct1), L.ptr(lvl1), L.ptr(cnt), C_, 19, iters,
                                                  gk.ctypes.data_as(C.c_void_p), L.ptr(A), st))
            else:
                base, cur = None, nl
                for it in range(iters):
                    Ai = net(a, cur, oct1, lvl1, cnt, 4)
                    if base is None:
                        base = Ai
                    else:
                        nb = empty(B, C_, 4)
                        L.check(lib.ag_mat2_compose(L.ptr(Ai), L.ptr(base), L.ptr(nb), n, st))
                        base = nb
                    if it != iters - 1:
                        cur = empty(B, C_, 2, 3)
                        L.check(lib.ag_lafs_left_multiply(L.ptr(base), L.ptr(nl), L.ptr(cur), n, st))
                A = base
            resp = torch.arange(C_, dtype=torch.float32, device=DEV).repeat(B, 1).contiguous()
            src_f, lafs2 = empty(B, C_), empty(B, C_, 2, 3)
            oct2, lvl2, cnt2 = empty(B, C_, dtype=torch.int32), empty(B, C_, dtype=torch.int32), empty(B, dtype=torch.int32)
            L.check(lib.ag_affine_shape_filter_all(L.ptr(A), L.ptr(resp), L.ptr(nl), L.ptr(oct1), L.ptr(lvl1), L.ptr(cnt), B, C_,
                                                   L.ptr(src_f), L.ptr(lafs2), L.ptr(oct2), L.ptr(lvl2), L.ptr(cnt2), st))
            cnt = cnt2
            src = src_f.to(torch.int32)
        else:
            lafs2, oct2, lvl2 = nl, oct1, lvl1
        if ori == "orinet":
            R = net(o, lafs2, oct2, lvl2, cnt, 4)
            L.check(lib.ag_lafs_apply_rotation(L.ptr(lafs2), L.ptr(R), n, st))
        elif ori == "histogram":
            gk = np.zeros((19, 19), np.float32)
            L.check(lib.ag_circular_gauss_kernel(19, 0.0, gk.ctypes.data_as(C.c_void_p)))
            gk = (gk * np.float32(10.0)).astype(np.float32)
            R = empty(B, C_, 4)
            L.check(lib.ag_debug_orientation_hist_pyr(plan, L.ptr(pyr), L.ptr(lafs2), L.ptr(oct2), L.ptr(lvl2), L.ptr(cnt), C_, 19,
                                                      gk.ctypes.data_as(C.c_void_p), L.ptr(R), st))
            L.check(lib.ag_lafs_apply_rotation(L.ptr(lafs2), L.ptr(R), n, st))
        dl = scale(lafs2, ms, float(W_), float(H))
    dps = int(desc[4:]) if desc.startswith("sift") else 32
    oct3, lvl3 = level(dl, dps)
    nl3 = scale(dl, na, nx, ny)
    if desc.startswith("sift"):
        d = empty(B, C_, 128)
        L.check(lib.ag_sift_describe_pyr(plan, L.ptr(pyr), L.ptr(nl3), L.ptr(oct3), L.ptr(lvl3), L.ptr(cnt), C_, dps, 0.2, L.ptr(d), st))
    else:
        d = net(h, nl3, oct3, lvl3, cnt, 128)
    return dl, src, d, cnt


@pytest.mark.parametrize("mode", MODES, ids=lambda m: "%s%s-%s-%s" % (m[0], m[1], m[2], m[3]))
def test_composition_of_existing_entry_points_bit_for_bit(L, nets, mode):
    shape, iters, ori, desc = mode
    img = crop_img()
    imgs = torch.cat([img, torch.flip(img, dims=[2])], 0).to(DEV).contiguous()
    B, H, W_, C_ = 2, img.size(2), img.size(3), 400
    lafs_in = torch.stack([random_keypoints(C_, H, W_, 7), random_keypoints(C_, H, W_, 8)]).to(DEV).contiguous()
    counts = torch.tensor([C_, 271], dtype=torch.int32, device=DEV)
    g = given_pipe(B, H, W_, nets, shape, iters, ori, desc, C_)
    gl, gs, gd, gc = g.run(imgs, lafs_in, counts)
    plan = L.lib().ag_pipeline_plan(g._h)
    pyr = torch.empty(plan.contents.total_floats, dtype=torch.float32, device=DEV)
    L.check(L.lib().ag_pyramid_build(plan, L.ptr(imgs), L.ptr(pyr), L.stream_ptr()))
    dl, src, d, cnt = composition(L, nets, plan, pyr, lafs_in, counts, C_, shape, iters, ori, desc, H, W_)
    torch.cuda.synchronize()
    assert torch.equal(gc, cnt)
    for b in range(B):
        m = int(cnt[b])
        assert m > 50
        assert torch.equal(gs[b, :m], src[b, :m])
        assert bits_equal(gl[b, :m], dl[b, :m]) and bits_equal(gd[b, :m], d[b, :m])
        assert (gl[b, m:] == SENTINEL).all() and (gd[b, m:] == SENTINEL).all() and (gs[b, m:] == ISENT).all()
    if shape is not None:
        assert int(cnt[0]) < C_          # the boundary test drops the keypoints across the border


# ---- 3. against the oracle on graf 1024x768 -----------------------------------------------------------------------------------------------
def test_against_the_oracle_graf_1024(L, nets):
    """Upright keypoints of graf 1024x768 (the detector without a shape or orientation step) -> AffNet x 1 + OriNet + HardNet: the
    oracle's survivors (except rows on the eigenvalue test's knife edge), LAFs within 1e-3 of the scale, descriptors within 1e-3."""
    from affnet_b200.pipeline import DetectDescribePipeline
    img = graf_1024()
    H, W_ = img.size(2), img.size(3)
    a, o, h = nets
    det = DetectDescribePipeline(1, H, W_, None, h, None, num_features=1000, do_ori=False, num_Baum_iters=0)
    lafs, _, _, cnt = det.run(img.to(DEV).contiguous())
    n = int(cnt[0])
    g = given_pipe(1, H, W_, nets, "affnet", 1, "orinet", "hardnet", 1000)
    gl, gs, gd, gc = g.run(img.to(DEV).contiguous(), lafs, cnt)
    torch.cuda.synchronize()
    m = int(gc[0])
    torch.set_num_threads(min(16, torch.get_num_threads()))
    oL, osrc, od, st = G.describe_given(img, lafs[0, :n].cpu(), "affnet", 1, W["affnet"], "orinet", W["orinet"], W["hardnet"])
    edge = G.knife_edge(st["debug"]["aff"]["base_A"])
    mine = gs[0, :m].cpu().tolist()
    diff = set(mine) ^ set(osrc.tolist())
    print("\n%d keypoints, %d survivors (oracle %d), disagreements %s" % (n, m, osrc.numel(), sorted(diff)))
    assert all(bool(edge[i]) for i in diff) and len(diff) <= max(2, n // 200)
    common = sorted(set(mine) & set(osrc.tolist()))
    ig = torch.tensor([mine.index(i) for i in common])
    io = torch.tensor([osrc.tolist().index(i) for i in common])
    dL = gl[0, :m].cpu()[ig]
    s = (oL[io][:, 0, 0] * oL[io][:, 1, 1] - oL[io][:, 0, 1] * oL[io][:, 1, 0]).abs().sqrt()
    eL = ((dL - oL[io]).abs().amax(dim=(1, 2)) / s)
    dd = (gd[0, :m].cpu()[ig] - od[io]).abs().amax(dim=1)
    print("LAF error max %.2e, descriptor max %.2e" % (eL.max(), dd.max()))
    assert float((eL < TOL).float().mean()) >= 0.995 and float((dd < TOL).float().mean()) >= 0.995


# ---- 4. rows and counts -------------------------------------------------------------------------------------------------------------------
def test_ragged_counts_and_poison(L, nets):
    """Counts C, a ragged count, 0, -1 and C + 1: the last two give -1 and no row written; rows at or beyond every count keep the
    sentinel.  A valid image's rows equal a B = 1 run on that image alone."""
    img = crop_img()
    H, W_, C_ = img.size(2), img.size(3), 300
    imgs = torch.cat([img] * 5, 0).to(DEV).contiguous()
    lafs_in = torch.stack([random_keypoints(C_, H, W_, s) for s in range(5)]).to(DEV).contiguous()
    counts = torch.tensor([C_, 17, 0, -1, C_ + 1], dtype=torch.int32, device=DEV)
    g = given_pipe(5, H, W_, nets, "affnet", 1, "orinet", "hardnet", C_)
    gl, gs, gd, gc = g.run(imgs, lafs_in, counts)
    one = given_pipe(1, H, W_, nets, "affnet", 1, "orinet", "hardnet", C_)
    torch.cuda.synchronize()
    c = gc.cpu().tolist()
    assert c[2] == 0 and c[3] == -1 and c[4] == -1 and 0 < c[0] < C_ and 0 < c[1] <= 17
    for b in range(5):
        m = max(c[b], 0)
        assert (gl[b, m:] == SENTINEL).all() and (gd[b, m:] == SENTINEL).all() and (gs[b, m:] == ISENT).all()
    for b in (0, 1):
        ol, os_, od, oc = one.run(imgs[b:b + 1], lafs_in[b:b + 1], counts[b:b + 1])
        torch.cuda.synchronize()
        m = c[b]
        assert int(oc[0]) == m and torch.equal(os_[0, :m], gs[b, :m])
        assert bits_equal(ol[0, :m], gl[b, :m]) and bits_equal(od[0, :m], gd[b, :m])
    # keypoints entirely outside the image never survive the boundary test
    inside = lafs_in[0, gs[0, :c[0]].long()]
    assert ((inside[:, :, 2] >= 0).all() and (inside[:, 0, 2] <= W_).all() and (inside[:, 1, 2] <= H).all())


def test_capacity_above_the_sort_limit(L, nets):
    """C = 20000 rows per image (above the top-K kernels' 16384), Baumberg + histogram + SIFT: as the composition of the entry points,
    with the rows beyond the counts untouched."""
    img = crop_img()
    H, W_, C_ = img.size(2), img.size(3), 20000
    imgs = torch.cat([img, img], 0).to(DEV).contiguous()
    lafs_in = torch.stack([random_keypoints(C_, H, W_, 11), random_keypoints(C_, H, W_, 12)]).to(DEV).contiguous()
    counts = torch.tensor([C_, 19000], dtype=torch.int32, device=DEV)
    g = given_pipe(2, H, W_, nets, "baumberg", 1, "histogram", "sift32", C_)
    gl, gs, gd, gc = g.run(imgs, lafs_in, counts)
    plan = L.lib().ag_pipeline_plan(g._h)
    pyr = torch.empty(plan.contents.total_floats, dtype=torch.float32, device=DEV)
    L.check(L.lib().ag_pyramid_build(plan, L.ptr(imgs), L.ptr(pyr), L.stream_ptr()))
    dl, src, d, cnt = composition(L, nets, plan, pyr, lafs_in, counts, C_, "baumberg", 1, "histogram", "sift32", H, W_)
    torch.cuda.synchronize()
    assert torch.equal(gc, cnt) and int(gc[0]) > C_ // 2
    for b in range(2):
        m = int(cnt[b])
        assert torch.equal(gs[b, :m], src[b, :m]) and bits_equal(gl[b, :m], dl[b, :m]) and bits_equal(gd[b, :m], d[b, :m])
        assert (gd[b, m:] == SENTINEL).all() and (gs[b, m:] == ISENT).all()


# ---- 5. ag_ells_to_lafs -------------------------------------------------------------------------------------------------------------------
def test_ells_to_lafs_bit_for_bit_and_round_trip(L):
    from affnet_b200.LAF import LAFs2ellT, ells2LAFsT
    z = gold("given.npz")
    ell = torch.from_numpy(z["ell_in"]).to(DEV)
    out = ells2LAFsT(ell).cpu().numpy()
    ref = G.ells_to_lafs(z["ell_in"])
    assert np.array_equal(np.isnan(out), np.isnan(ref))
    assert np.array_equal(np.nan_to_num(out, nan=0.0).view(np.uint32), np.nan_to_num(ref, nan=0.0).view(np.uint32))
    # round trip through ag_lafs_to_ell, bounded in float64
    back = LAFs2ellT(ells2LAFsT(ell)).cpu().double().numpy()
    e = z["ell_in"].astype(np.float64)
    fin = ~np.isnan(back).any(axis=1) & ~np.isnan(out).any(axis=(1, 2))
    assert fin.mean() > 0.98
    M = lambda r: np.stack([r[:, 2], r[:, 3], r[:, 3], r[:, 4]], 1).reshape(-1, 2, 2)
    err = np.abs(M(back[fin]) - M(e[fin])).max(axis=(1, 2)) / np.abs(M(e[fin])).max(axis=(1, 2))
    print("\nround trip: %d rows, relative error median %.2e max %.2e" % (fin.sum(), np.median(err), err.max()))
    assert np.quantile(err, 0.95) < 1e-4 and np.array_equal(back[fin, :2], e[fin, :2])


# ---- 6. one CUDA graph from images and keypoints to verified matches ----------------------------------------------------------------------
def test_one_graph_given_match_verify(L, nets):
    """graf img1 and img6 with their upright detections: the given pipeline, match_snn_pairs and find_homography_pairs /
    gt_correspondences_pairs captured in one CUDA graph; its replay equals the eager run bit for bit."""
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.ReprojectionStuff import find_homography_pairs, gt_correspondences_pairs
    zm = gold("graf_match.npz")
    imgs = torch.cat([gray_from_rgb(gold("graf_full.npz")["rgb"]), gray_from_rgb(zm["rgb6"])], 0).to(DEV).contiguous()
    H1to6 = torch.from_numpy(zm["H1to6"]).float().to(DEV)
    B, H, W_, C_ = 2, imgs.size(2), imgs.size(3), 2000
    a, o, h = nets
    det = DetectDescribePipeline(B, H, W_, None, h, None, num_features=C_, do_ori=False, num_Baum_iters=0)
    lafs, _, _, cnt = det.run(imgs)
    lafs, cnt = lafs.clone(), cnt.clone()
    g = given_pipe(B, H, W_, nets, "affnet", 1, "orinet", "hardnet", C_)

    def step():
        gl, gs, gd, gc = g.run(imgs, lafs, cnt)
        tent, ntent, _, _ = match_snn_pairs(gd[0:1], gc[0:1], gd[1:2], gc[1:2])
        Hh, inl, ninl, _ = find_homography_pairs(gl[0:1], tent, ntent, gl[1:2])
        tr, ntrue, _, _ = gt_correspondences_pairs(gl[0:1], tent, ntent, H1to6, gl[1:2])
        return [gl, gs, gd, gc, tent, ntent, Hh, inl, ninl, tr, ntrue]

    eager = [t.clone() for t in step()]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        outs = step()
    for t in outs:
        if t.dtype == torch.float32:
            t.fill_(SENTINEL)
    gr.replay()
    torch.cuda.synchronize()
    gl, gs, gd, gc, tent, ntent, Hh, inl, ninl, tr, ntrue = outs
    e = eager
    assert torch.equal(gc, e[3]) and torch.equal(ntent, e[5]) and torch.equal(ninl, e[8]) and torch.equal(ntrue, e[10])
    for b in range(B):
        m = int(gc[b])
        assert bits_equal(gl[b, :m], e[0][b, :m]) and torch.equal(gs[b, :m], e[1][b, :m]) and bits_equal(gd[b, :m], e[2][b, :m])
    nt, nv = int(ntent[0]), int(ntrue[0])
    assert torch.equal(tent[0, :nt], e[4][0, :nt]) and bits_equal(Hh, e[6]) and torch.equal(inl[0, :nt], e[7][0, :nt])
    assert torch.equal(tr[0, :nv], e[9][0, :nv])
    print("\ngraf 1-6 given: %d / %d keypoints, %d tentatives, %d inliers, %d true" % (int(gc[0]), int(gc[1]), nt, int(ninl[0]), nv))
    assert nt > 20 and nv > 10
