"""Shared test helpers (fixtures loading, keypoint matching)."""
import os

import numpy as np
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def gold(name):
    return np.load(os.path.join(GOLD, name))


def load_weights():
    """-> dict(affnet=sd, orinet=sd, hardnet=sd) of float32 torch tensors (checkpoint key names)."""
    z = gold("weights.npz")
    out = {"affnet": {}, "orinet": {}, "hardnet": {}}
    for k in z.files:
        net, key = k.split("/", 1)
        out[net][key] = torch.from_numpy(z[k])
    return out


def gray_from_rgb(rgb):
    """hesaffnet.py:35-39: mean over RGB -> float32 [1,1,H,W]."""
    return torch.from_numpy(np.mean(rgb, axis=2).astype(np.float32)).view(1, 1, rgb.shape[0], rgb.shape[1])


def match_keypoints(LA, LB, tol_px=0.05):
    """Greedy one-to-one matching of LAF centres. Returns (idxA, idxB) of matched pairs."""
    a = LA[:, :, 2].double().numpy(); b = LB[:, :, 2].double().numpy()
    from scipy.spatial import cKDTree
    tree = cKDTree(b)
    d, j = tree.query(a, k=1)
    ok = d <= tol_px
    ia = np.nonzero(ok)[0]; ib = j[ok]
    # scale check disambiguates same-centre detections from different levels
    keep = []
    used = set()
    for x, y in zip(ia, ib):
        if y in used:
            continue
        sa = abs(np.linalg.det(LA[x, :, :2].double().numpy())) ** 0.5
        sb = abs(np.linalg.det(LB[y, :, :2].double().numpy())) ** 0.5
        if abs(sa - sb) <= 0.05 * max(sa, 1.0):
            keep.append((x, y)); used.add(y)
    if not keep:
        return np.zeros(0, int), np.zeros(0, int)
    k = np.array(keep)
    return k[:, 0], k[:, 1]


def laf_rel_errors(LA, LB):
    """Parity contract for matched LAFs (SURVEY Q7 ii, north_star 1e-3): errors RELATIVE to the LAF scale s = sqrt(|det A|) of the
    first argument.  Returns (max |dA| / s, max |dcentre| / s) over the rows."""
    A, B = LA.double(), LB.double()
    s = (A[:, 0, 0] * A[:, 1, 1] - A[:, 0, 1] * A[:, 1, 0]).abs().sqrt().clamp_min(1e-12)
    eA = ((A[:, :, :2] - B[:, :, :2]).abs().amax(dim=(1, 2)) / s).max().item()
    ec = ((A[:, :, 2] - B[:, :, 2]).abs().amax(dim=1) / s).max().item()
    return eA, ec


def parity_report(oL, odesc, dL, desc, tag=""):
    """Match keypoints of the oracle (oL, odesc) and the CUDA path (dL, desc); returns dict(matched, n, eA, ec, dd) and prints it."""
    ia, ib = match_keypoints(oL, dL)
    eA, ec = laf_rel_errors(oL[ia], dL[ib]) if len(ia) else (float("inf"), float("inf"))
    dd = (odesc[ia] - desc[ib]).abs().max().item() if len(ia) else float("inf")
    out = dict(matched=len(ia), n=int(oL.shape[0]), n_ours=int(dL.shape[0]), eA=eA, ec=ec, dd=dd)
    print("\n%s: matched %d/%d (ours %d)  max|dA|/scale %.2e  max|dcentre|/scale %.2e  max|ddesc| %.2e" % (tag, out["matched"], out["n"], out["n_ours"], eA, ec, dd))
    return out


TOL = 1e-3     # north_star: LAF parameters (relative to the LAF scale) and HardNet descriptors within 1e-3

# ---- direct calls of the net entry points with row counts and a caller-owned workspace -------------------------------------------
POISON_NAN, POISON_INF = 0xFFFF, 0x7C00    # 16-bit words a workspace is filled with: all-ones bytes (NaN in fp16 and fp32), fp16 +Inf
SENTINEL = -12345.0                        # output rows a call must not write keep this value


def poisoned(nbytes, word, device="cuda"):
    """A device buffer of `nbytes` (even) bytes whose every 16-bit word is `word`, or uninitialised when word is None."""
    buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
    if word is not None:
        buf.view(torch.int16).fill_(word - 0x10000 if word >= 0x8000 else word)
    return buf


def row_valid(n, group, counts):
    """Row validity of the C ABI: row i is valid when i % group < counts[i // group] (counts None: every row).  -> bool [n]."""
    if counts is None:
        return torch.ones(n, dtype=torch.bool)
    i = torch.arange(n)
    return (i % group) < torch.as_tensor(counts, dtype=torch.int64)[i // group]


def net_forward_rows(L, net, patches, counts=None, group=0, ws_word=None):
    """ag_affnet_forward / ag_orinet_forward / ag_hardnet_forward called directly on CUDA patches [n,1,32,32] with the net's current
    engine: `counts` (list of ints, one per group of `group` rows; None = NULL count array) is uploaded as the device int32 array, the
    workspace of ag_net_workspace_bytes(kind, n) bytes is owned here and filled with `ws_word` (see poisoned), and the outputs start
    as SENTINEL.  Returns (out, angle): out [n,2,2] (AffNet, OriNet) or [n,128] (HardNet); angle [n] for OriNet (both outputs are
    requested), else None."""
    lib = L.lib()
    n = patches.size(0)
    P = patches.to("cuda", torch.float32).contiguous()
    nbytes = lib.ag_net_workspace_bytes(net.KIND, n)
    ws = poisoned(nbytes, ws_word)
    cnt = None if counts is None else torch.tensor(counts, dtype=torch.int32, device="cuda")
    out = torch.full((n, 128) if net.KIND == L.NET_HARDNET else (n, 2, 2), SENTINEL, device="cuda")
    angle = torch.full((n,), SENTINEL, device="cuda") if net.KIND == L.NET_ORINET else None
    if net.KIND == L.NET_AFFNET:
        rc = lib.ag_affnet_forward(net.handle(), L.ptr(P), n, L.ptr(cnt), group, L.ptr(out), L.ptr(ws), nbytes, L.stream_ptr())
    elif net.KIND == L.NET_ORINET:
        rc = lib.ag_orinet_forward(net.handle(), L.ptr(P), n, L.ptr(cnt), group, L.ptr(out), L.ptr(angle), L.ptr(ws), nbytes, L.stream_ptr())
    else:
        rc = lib.ag_hardnet_forward(net.handle(), L.ptr(P), n, L.ptr(cnt), group, L.ptr(out), L.ptr(ws), nbytes, L.stream_ptr())
    L.check(rc)
    torch.cuda.synchronize()
    return out, angle


def net_forward_pyr(L, net, plan, pyr, lafs, octs, lvls, counts, cap, ws_word=None):
    """ag_net_forward_pyr over a pyramid (plan, flat buffer) with LAFs [B*cap,2,3] normalised, octave / level indices [B*cap] and the
    per-image counts (list of B ints; None = NULL), over a workspace filled with `ws_word`, into an output prefilled with SENTINEL.
    Returns (rc, out): the call's return code is handed back unchecked."""
    import ctypes as C
    lib = L.lib()
    n = plan.B * cap
    nbytes = lib.ag_net_workspace_bytes(net.KIND, n)
    ws = poisoned(nbytes, ws_word)
    cnt = None if counts is None else torch.tensor(counts, dtype=torch.int32, device="cuda")
    d = lambda t, dt: t.to("cuda", dt).contiguous()  # noqa: E731
    dl, do, dv = d(lafs, torch.float32), d(octs, torch.int32), d(lvls, torch.int32)
    out = torch.full((n, 128) if net.KIND == L.NET_HARDNET else (n, 2, 2), SENTINEL, device="cuda")
    rc = lib.ag_net_forward_pyr(net.handle(), C.byref(plan), L.ptr(pyr), L.ptr(dl), L.ptr(do), L.ptr(dv), L.ptr(cnt), cap, L.ptr(out),
                                L.ptr(ws), nbytes, L.stream_ptr())
    torch.cuda.synchronize()
    return rc, out


def synthetic_image(H, W, seed):
    """SURVEY.md §8(d) config 3 input: U[0,255) noise blurred with sigma=2 (separable, replicate border), stretched to 0..255.
    Bit-identical to oracle/affnet_oracle.py::synthetic_image (tests/test_lib_cpu.py checks it); lives here so that bench.py's
    product arm generates its inputs without importing the oracle."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(1, 1, H, W, generator=g) * 255.0
    sigma = 2.0
    k = int(2.0 * 3.0 * sigma + 1.0)
    if k % 2 == 0:
        k += 1
    half = k / 2.0
    xs = np.linspace(-half, half, k)
    e = np.exp(-(xs * xs) / (2.0 * sigma * sigma))
    k1 = torch.from_numpy((e / e.sum()).astype(np.float32))
    x = F.conv2d(F.pad(x, (k // 2, k // 2, 0, 0), "replicate"), k1.view(1, 1, 1, k))
    x = F.conv2d(F.pad(x, (0, 0, k // 2, k // 2), "replicate"), k1.view(1, 1, k, 1))
    x = (x - x.min()) / (x.max() - x.min()) * 255.0
    return x.contiguous()


def orientation_boundary_shares(patches, tol_bins=1e-4, num_bins=36):
    """Hand-crafted orientation (HandCraftedModules.py:168-190) accumulates only the LOWER-bin weight (1 - frac) * magnitude of every pixel,
    so a pixel whose gradient orientation lies on a bin boundary moves its whole weight between two bins under an arbitrarily small change of
    the patch.  For patches [n,1,PS,PS] returns (margin [n], share [n]): the relative margin between the two best smoothed bins, and the
    largest weight - relative to the best bin - among the pixels within `tol_bins` of a boundary (0 if none).  share > margin means: an
    epsilon perturbation can legitimately change the arg-max bin although the two best bins are not tied."""
    import math

    import torch.nn.functional as F

    import affnet_oracle as O
    PS = patches.size(2)
    xp = F.pad(patches, (1, 1, 0, 0), "replicate")
    gx = 0.5 * xp[:, :, :, :-2] - 0.5 * xp[:, :, :, 2:]
    yp = F.pad(patches, (0, 0, 1, 1), "replicate")
    gy = 0.5 * yp[:, :, :-2, :] - 0.5 * yp[:, :, 2:, :]
    gk = 10.0 * torch.from_numpy(O.circular_gauss_kernel(PS).astype(np.float32))
    mag = torch.sqrt(gx * gx + gy * gy + 1e-10) * gk
    o_big = float(num_bins) * (torch.atan2(gy, gx) + math.pi) / (2.0 * math.pi)
    frac = o_big - torch.floor(o_big)
    dist = torch.minimum(frac, 1.0 - frac).flatten(1)
    sm = O.orientation_hist_bins(patches, num_bins)
    top = sm.topk(2, dim=1).values
    margin = (top[:, 0] - top[:, 1]) / top[:, 0]
    w = (mag.flatten(1) / float(PS * PS)) / top[:, :1]
    share = torch.where(dist < tol_bins, w, torch.zeros_like(w)).amax(dim=1)
    return margin, share


# ---- detector stage: pyramids no blur would produce, and the oracle's keypoints in the selection's order ----------------------------
SEQ_PIX_BITS = 27                           # candidate seq = (level slot << 27) | flat pixel index (include/affnet_b200.h)
ADV_H = ADV_W = 40                          # adversarial pyramids: plan(40, 40, border 5) has octaves 40x40 and 20x20


def _bump_levels(g, n, h, w, lo, span, max_sigma):
    yy, xx = torch.meshgrid(torch.arange(h).float(), torch.arange(w).float(), indexing="ij")
    levels = []
    for _ in range(n):
        k = int(torch.randint(0, 3, (1,), generator=g))
        img = torch.full((h, w), 10.0)
        for _ in range(k):
            cy, cx = (torch.rand(2, generator=g) * span + lo).tolist()
            s = float(torch.rand(1, generator=g) * (max_sigma - 1.0) + 1.0)
            a = float(torch.rand(1, generator=g) * 60 + 1)
            img += a * torch.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * s * s))
        levels.append(img.view(1, 1, h, w))
    return levels


def adversarial_pyramid(seed, nlevels=3):
    """A pyramid for plan(B, 40, 40, nlevels, 1.6, 5) that drives the level-drop rule: every level of octave 0 is a constant 10 plus 0-2
    Gaussian bumps (sigma 1-3, amplitude 1-61, centres in [8, 32)), so levels with 0, 1 or 2 positive maxima, negative masked responses
    and wrapping uint8 octave maps all occur.  Octave 1 (20x20) is constant or gets its own bumps.  -> pyr[o][l] float32 [1,1,h,w]."""
    g = torch.Generator().manual_seed(seed)
    n = nlevels + 2
    oct0 = _bump_levels(g, n, ADV_H, ADV_W, 8.0, 24.0, 3.0)
    h1, w1 = (ADV_H + 1) // 2, (ADV_W + 1) // 2
    if int(torch.randint(0, 2, (1,), generator=g)):
        oct1 = [torch.full((1, 1, h1, w1), 10.0) for _ in range(n)]
    else:
        oct1 = _bump_levels(g, n, h1, w1, 4.0, 12.0, 2.0)
    return [oct0, oct1]


def detector_level_stats(octave, sigmas, mrSize, th=0.0):
    """Per detection level of one octave, from the oracle's primitives (HandCraftedModules.py:240-263): (n_pos, accepted, has negative
    masked responses, octave map wrapped).  n_pos <= 1 drops the level; 'wrapped' means some pixel's uint8 map value came out below
    the float sum it truncates (Q4)."""
    import affnet_oracle as O
    h, w = octave[0].size(2), octave[0].size(3)
    maps = [torch.clamp(O.hessian_response(octave[l], sigmas[l]) - th, min=0) for l in range(len(octave))]
    om = np.zeros((h, w), np.uint8)
    b = int(mrSize)
    out = []
    for l in range(1, len(octave) - 1):
        nm = O.nms3d_mask(maps[l - 1], maps[l], maps[l + 1]).clone()
        if b < w and b < h:
            nm[:, :, :b, :] = 0; nm[:, :, h - b:, :] = 0; nm[:, :, :, :b] = 0; nm[:, :, :, w - b:] = 0
        else:
            nm = nm * 0
        nm = nm * (1.0 - torch.from_numpy(om.astype(np.float32)).view(1, 1, h, w))
        n_pos = int((nm > 0).sum())
        neg = bool((nm < 0).any())
        r, _, om2, _ = O.nms3d_and_compose(maps[l - 1], maps[l], maps[l + 1], 0, om, sigmas[l - 1:l + 2], mrSize)
        wrapped = r is not None and bool((om2.astype(np.float64) < np.trunc((om.astype(np.float64) + nm.numpy().reshape(h, w)).clip(0))).any())
        out.append((n_pos, r is not None, neg, wrapped))
        om = om2
    return out


def mixed_batch(h, w, seed):
    """Two textured images around a constant one (which has no keypoint)."""
    return torch.cat([synthetic_image(h, w, seed), torch.full((1, 1, h, w), 77.0), synthetic_image(h, w, seed + 1)])


def plan_sigmas(plan):
    return [[plan.sigma[o][l] for l in range(plan.n_levels)] for o in range(plan.n_octaves)]


def flat_pyramid(plan, pyrs, device="cuda"):
    """pyrs[b][o][l] ([1,1,h_o,w_o] or [h_o,w_o]) -> the plan's device buffer: image b of level (o, l) at level_offset[o][l] + b*h_o*w_o."""
    buf = torch.zeros(plan.total_floats, dtype=torch.float32)
    for b, pyr in enumerate(pyrs):
        for o in range(plan.n_octaves):
            n = plan.h[o] * plan.w[o]
            for l in range(plan.n_levels):
                off = plan.level_offset[o][l] + b * n
                buf[off:off + n] = pyr[o][l].reshape(-1)
    return buf.to(device)


def gpu_pyramids(L, imgs, nlevels=3, border=5):
    """The GPU blur's pyramid of imgs [B,1,H,W] -> (plan, device buffer, per-image CPU copies pyrs[b][o][l] [1,1,h,w])."""
    from affnet_b200.HandCraftedModules import ScalePyramid
    plan, buf = ScalePyramid(nlevels, 1.6, border).build(imgs.to("cuda").contiguous())
    views, _, _ = ScalePyramid.views(plan, buf)
    pyrs = [[[lv[b:b + 1].cpu() for lv in octave] for octave in views] for b in range(plan.B)]
    return plan, buf, pyrs


class Detector:
    """ag_detect once over a workspace of `cap` candidates per image; select() calls ag_select_keypoints and select_all()
    ag_select_all_keypoints into sentinel-filled outputs."""

    def __init__(self, L, plan, buf, th=0.0, mr=5.192, cap=None):
        import ctypes as C
        self.C, self.L, self.lib, self.plan = C, L, L.lib(), plan
        self.cap = cap or max(plan.H * plan.W // 4, 4096)
        self.ws_buf = torch.full((self.lib.ag_detect_ws_bytes(C.byref(plan), self.cap),), 0xFF, dtype=torch.uint8, device="cuda")
        self.ws = L.DetectWs()
        L.check(self.lib.ag_detect_ws_carve(C.byref(plan), self.cap, L.ptr(self.ws_buf), C.byref(self.ws)))
        L.check(self.lib.ag_detect(C.byref(plan), L.ptr(buf), float(th), int(mr), C.byref(self.ws), L.stream_ptr()))

    def cand_counts(self):
        off = self.ws.d_cand_count - self.ws_buf.data_ptr()
        return self.ws_buf[off:off + 4 * self.plan.B].view(torch.int32).cpu()

    def _outputs(self, cap):
        B, isent = self.plan.B, int(SENTINEL)
        return (torch.full((B, cap), SENTINEL, device="cuda"), torch.full((B, cap, 2, 3), SENTINEL, device="cuda"),
                torch.full((B, cap), isent, dtype=torch.int32, device="cuda"), torch.full((B, cap), isent, dtype=torch.int32, device="cuda"),
                torch.full((B,), isent, dtype=torch.int32, device="cuda"))

    def select(self, nf, out_cap=None, a_scale=1.0):
        """-> (rc, (resp [B,out_cap], lafs [B,out_cap,2,3], oct, lvl, count [B])) on the CPU."""
        C, L = self.C, self.L
        cap = out_cap or nf
        out = self._outputs(cap)
        rc = self.lib.ag_select_keypoints(C.byref(self.plan), C.byref(self.ws), int(nf), float(a_scale), cap, *[L.ptr(t) for t in out],
                                          L.stream_ptr())
        torch.cuda.synchronize()
        return rc, tuple(t.cpu() for t in out)

    def checked_select(self, nf, out_cap=None, a_scale=1.0):
        rc, out = self.select(nf, out_cap, a_scale)
        self.L.check(rc)
        return out

    def select_all(self, out_cap, a_scale=1.0):
        """ag_select_all_keypoints (every candidate of the accepted levels, seq order) -> the outputs of select()."""
        C, L = self.C, self.L
        nbytes = self.lib.ag_select_all_workspace_bytes(C.byref(self.plan), self.cap)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        out = self._outputs(out_cap)
        L.check(self.lib.ag_select_all_keypoints(C.byref(self.plan), C.byref(self.ws), float(a_scale), out_cap, L.ptr(scratch), nbytes,
                                                 *[L.ptr(t) for t in out], L.stream_ptr()))
        torch.cuda.synchronize()
        return tuple(t.cpu() for t in out)


class OracleCandidates:
    """Every keypoint the oracle emits for one image before its global top-k (num_features <= 0: per-level raster order, octave after
    octave, level after level), with each one's seq; select(nf) applies the selection rule the C ABI documents: the top nf by (response
    descending, seq ascending) when more than nf remain or a level was trimmed, otherwise all in seq order.  An image without an accepted
    level has no candidates (the oracle, like the reference, raises from torch.cat there)."""

    def __init__(self, pyr, sigmas, mrSize, th=0.0):
        import affnet_oracle as O
        self.pyr, self.sigmas, self.mrSize, self.th = pyr, sigmas, mrSize, th
        n_det = len(pyr[0]) - 2
        try:
            self.resp, self.lafs, self.oct, self.lvl, dump = O.multi_scale_detector(pyr, sigmas, 0, mrSize, th=th, return_levels=True)
        except ValueError:                  # torch.cat of an empty list: no level of any octave was accepted
            self.resp, self.lafs, dump = torch.zeros(0), torch.zeros(0, 2, 3), [(o, l, None, None) for o in range(len(pyr)) for l in range(1, n_det + 1)]
            self.oct = self.lvl = torch.zeros(0)
        self.accepted = {(o, l - 1): idxs is not None for (o, l, idxs, _) in dump}
        self.n_pos = [int((r > 0).sum()) for (_, _, idxs, r) in dump if idxs is not None]
        self.seq = torch.cat([((o * n_det + l - 1) << SEQ_PIX_BITS) + idxs for (o, l, idxs, _) in dump if idxs is not None] or [torch.zeros(0, dtype=torch.int64)])
        self.total = self.resp.numel()

    def order(self, nf):
        trimmed = nf > 0 and any(nf < p for p in self.n_pos)
        if nf > 0 and (self.total > nf or trimmed):
            return np.lexsort((self.seq.numpy(), -self.resp.double().numpy()))[:nf], True
        return np.arange(self.total), False

    def select(self, nf):
        """-> (resp, lafs, oct, lvl, seq, sorted)."""
        idx, srt = self.order(nf)
        idx = torch.from_numpy(np.ascontiguousarray(idx)).long()
        return self.resp[idx], self.lafs[idx], self.oct[idx], self.lvl[idx], self.seq[idx], srt

    def check_against_oracle(self, nf):
        """select(nf) must be what O.multi_scale_detector(.., nf, ..) returns, up to the order of equal responses: the same values in the
        same order, and the same keypoint wherever the value is unique among all candidates.  Returns the number of tie groups that
        straddle the cut (some members selected, some not)."""
        import affnet_oracle as O
        r, la, po, lo = self.select(nf)[:4]
        try:
            r_o, L_o, p_o, l_o = O.multi_scale_detector(self.pyr, self.sigmas, nf, self.mrSize, th=self.th)
        except ValueError:
            r_o = L_o = p_o = l_o = None
        if self.total == 0:
            assert r_o is None
            return 0
        assert torch.equal(r, r_o), (nf, r.numel(), r_o.numel())
        vals, counts = torch.unique(self.resp, return_counts=True)
        multi = vals[counts > 1]
        uniq = ~torch.isin(r, multi)
        assert torch.equal(la[uniq], L_o[uniq]) and torch.equal(po[uniq], p_o[uniq]) and torch.equal(lo[uniq], l_o[uniq]), nf
        sel_vals, sel_counts = torch.unique(r, return_counts=True)
        all_counts = dict(zip(vals.tolist(), counts.tolist()))
        return sum(1 for v, c in zip(sel_vals.tolist(), sel_counts.tolist()) if all_counts[v] > c)
