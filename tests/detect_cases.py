"""Detector inputs aimed at the soft-argmax's edges (test infrastructure, not product): pyramids with isolated blobs on the seams of
the register kernel's 30-column strips and 48-row bands and at the image's edges and corners, pyramids scaled down by powers of two
(low contrast: the 1e-8 of den goes from negligible to dominant, and the responses become fp32 subnormals), and the reference's
golden detector rows with their candidates' (slot, pixel)."""
import torch

import affnet_oracle as O
from detect_restated import EPS_DEN, level_maps, windows
from helpers import SEQ_PIX_BITS, gold, gray_from_rgb, synthetic_image

WCOLS, WROWS = 30, 48                   # output columns per strip and rows per band of detect_rows_kernel
LOW_K = (0, 8, 12, 16, 20, 60, 66)      # low-contrast cases: the pyramid times 2^-k (exact), the responses times 2^-2k
SEAM_SHAPE = (100, 130)                 # octave 0 holds the band seam at rows 47 / 48 and 95 / 96, strip seams at 29 / 30 and 59 / 60
TINY = 2.0 ** -126                      # smallest normal fp32


def _blob_targets(h, w):
    """Blob centres on the strip and band seams, at the corners and on the four edges of an h x w octave."""
    pts = [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1), (0, w // 2), (h - 1, w // 3), (h // 2, 0), (h // 3, w - 1)]
    for x in range(WCOLS - 1, w, WCOLS):
        pts += [(min(h - 1, 20 + 7 * (x // WCOLS)), x), (min(h - 1, 40 + 9 * (x // WCOLS)), x + 1)]
    for y in range(WROWS - 1, h, WROWS):
        pts += [(y, min(w - 1, 15 + 11 * (y // WROWS))), (y + 1, min(w - 1, 45 + 13 * (y // WROWS)))]
    return pts


def seam_pyramid(sizes, nlevels, seed):
    """pyr[o][l] [1,1,h,w] for octave sizes `sizes`: a constant 10 plus one Gaussian blob per target of _blob_targets, with a
    per-level amplitude, width (sigma 0.8-1.6) and sub-pixel offset, so the maxima sit on the targets and their soft-argmax windows
    hold unequal levels."""
    g = torch.Generator().manual_seed(seed)
    pyr = []
    for (h, w) in sizes:
        yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
        pts = _blob_targets(h, w)
        amp = torch.rand(len(pts), generator=g) * 60 + 20
        levels = []
        for _ in range(nlevels + 2):
            img = torch.full((h, w), 10.0, dtype=torch.float64)
            jit = (torch.rand(len(pts), 2, generator=g) - 0.5) * 0.6
            sig = torch.rand(len(pts), generator=g) * 0.8 + 0.8
            for i, (cy, cx) in enumerate(pts):
                y0, x0 = cy + float(jit[i, 0]), cx + float(jit[i, 1])
                img += float(amp[i]) * torch.exp(-((yy - y0) ** 2 + (xx - x0) ** 2) / (2 * float(sig[i]) ** 2))
            levels.append(img.float().view(1, 1, h, w))
        pyr.append(levels)
    return pyr


def seam_case(nlevels=3, seed=3):
    """(sizes, sigmas, pyr) of the seam pyramid under the plan (1, 100, 130, nlevels, 1.6, 5)."""
    sizes, _, sig, _ = O.pyramid_plan(*SEAM_SHAPE, nlevels, 1.6, 5)
    return sizes, sig, seam_pyramid(sizes, nlevels, seed)


def low_contrast_case():
    """(sizes, sigmas, pyr) of a 160x200 synthetic image's oracle pyramid (plan (1, 160, 200, 3, 1.6, 5)), to be scaled by 2^-k."""
    sizes, _, sig, _ = O.pyramid_plan(160, 200, 3, 1.6, 5)
    pyr, sig2, _ = O.scale_pyramid(synthetic_image(160, 200, 7), 3, 1.6, 5)
    assert sig2 == sig
    return sizes, sig, pyr


def scaled(pyr, k):
    """pyr times 2^-k, level by level (exact for these values: the result stays a normal fp32)."""
    s = float(2.0 ** -k)
    return [[lv * s for lv in octave] for octave in pyr]


def reach(pyr, sigmas, seq, th=0.0):
    """What the candidates seq [n] of pyramid pyr reach, as counts: first / last output column of a strip (x mod 30 = 0 / 29), first /
    last row of a band (y mod 48 = 0 / 47), the four image edges, den = sum r below / above 1e-8, a subnormal tap in the window, and
    plateau maxima (another tap of the window at least the centre)."""
    n_det = len(pyr[0]) - 2
    seq = torch.as_tensor(seq).to(torch.int64)
    slot, pix = seq >> SEQ_PIX_BITS, seq & ((1 << SEQ_PIX_BITS) - 1)
    keys = ("strip_first", "strip_last", "band_first", "band_last", "top", "bottom", "left", "right", "den_below", "den_above",
            "subnormal", "plateau")
    out = dict.fromkeys(keys, 0)
    for o in range(len(pyr)):
        maps = None
        for k in range(n_det):
            sel = slot == o * n_det + k
            if not bool(sel.any()):
                continue
            maps = level_maps(pyr[o], sigmas[o], th) if maps is None else maps
            h, w = maps.shape[-2:]
            p = pix[sel]
            y, x = p // w, p % w
            R = windows(maps[k:k + 3], p).reshape(-1, 27).double()
            centre = R[:, 13].clone()
            others = R.clone()
            others[:, 13] = -1.0
            den = R.sum(1)
            for key, m in (("strip_first", x % WCOLS == 0), ("strip_last", x % WCOLS == WCOLS - 1), ("band_first", y % WROWS == 0),
                           ("band_last", y % WROWS == WROWS - 1), ("top", y == 0), ("bottom", y == h - 1), ("left", x == 0),
                           ("right", x == w - 1), ("den_below", den < EPS_DEN), ("den_above", den > EPS_DEN),
                           ("subnormal", ((R > 0) & (R < TINY)).any(1)), ("plateau", (others.max(1).values >= centre) & (centre != 0))):
                out[key] += int(m.sum())
    return out


def golden_rows():
    """The reference's detector rows with their candidates: [(name, pyr, sigmas, seq, reference LAFs, oracle LAFs, maps)].
    graf_crop.npz:det_LAFs is the global top-k of multi_scale_detector (whose index set and order the oracle reproduces);
    nms_q4.npz's rows are one level's candidates in raster order (all) or its top 20, on response maps given directly (as a
    three-level pyramid whose Hessian is bypassed: maps, else None)."""
    out = []
    z = gold("graf_crop.npz")
    pyr, sig, _ = O.scale_pyramid(gray_from_rgb(z["rgb"]))
    nf = int(1.5 * int(z["K"]))
    resp, lafs, _, _, dump = O.multi_scale_detector(pyr, sig, nf, 5.192, return_levels=True)
    n_det = len(pyr[0]) - 2
    r_cat = torch.cat([r for (_, _, i, r) in dump if i is not None])
    s_cat = torch.cat([((o * n_det + l - 1) << SEQ_PIX_BITS) + i for (o, l, i, _) in dump if i is not None])
    gi = torch.topk(r_cat, k=nf)[1] if 0 < nf < r_cat.numel() else torch.arange(r_cat.numel())
    assert torch.equal(r_cat[gi], resp) and torch.equal(resp, torch.from_numpy(z["det_resp"]))
    out.append(("graf_crop:det_LAFs", pyr, sig, s_cat[gi], torch.from_numpy(z["det_LAFs"]), lafs, None))
    q = gold("nms_q4.npz")
    maps = [torch.from_numpy(q[k]).view(1, 1, *q[k].shape) for k in ("low", "cur", "high")]
    for nf, tag in ((0, "all"), (20, "top20")):
        r, A, _, idxs = O.nms3d_and_compose(*maps, nf, q["omap"].copy(), list(q["scales"]), 5.192)
        assert torch.equal(r, torch.from_numpy(q[tag + "_resp"]))
        out.append(("nms_q4:%s_LAFs" % tag, [maps], [list(q["scales"])], idxs, torch.from_numpy(q[tag + "_LAFs"]), A,
                    [torch.cat([m[0] for m in maps])]))
    return out
