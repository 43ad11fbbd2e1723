"""Generates tests/golden/nonfinite.npz by running the UNMODIFIED reference (/root/reference, ducha-aiki/affnet) on CPU on images and
response maps that hold NaN, +inf and -inf values or overflow fp32:

    python tests/golden/make_golden_nonfinite.py

Images (float32, [1,1,h,w]): `base` is 64x80 smoothed noise in [0, 255] (three octaves at border 5), `small` 17x19 (one octave).
  nan_mid, nan_edge, nan_corner    one NaN pixel in the interior, on the top edge (read through the replicate pad), at the corner
  pinf, ninf                       one +inf / -inf pixel
  small_nan                        the 17x19 image with a NaN pixel
  oct1_nan                         `base`, with a NaN written into level 1 of octave 1 of the pyramid the detector builds (only
                                   that level sees it; the reference's ScalePyramid output is patched, nothing else).  It takes one
                                   of the two maxima of octave 1's second detection level, which is then dropped
  scale_<k>                        `base` * 2^k: the detector's response maps are finite at k = 54, 57 and 58 (where only the
                                   soft-argmax sums overflow, den included), hold the first inf responses at 60 (59 is finite),
                                   NaN survivors of the NMS at inf responses at 61 (0 * inf), and the first NaN from inf - inf at 63
Per image: img_<case>; hess_<case>_<i> = HessianResp()(img, sigma_i) for sigma in HESS_SIGMAS; det<K>_<case>_{resp,lafs,pyr,lvl} =
multiScaleDetector(img, K) (K = 0: keep-all, 50: top-K) with ScaleSpaceAffinePatchExtractor(mrSize=5.192, border=5, nlevels=3), empty
where the reference raises because no level was accepted.

Response-map cases of NMS3dAndComposeA(w, h, border=5, mrSize=5.192) (nms_<case>_{low,cur,high,omap,scales} in,
nms_<case>_{resp,lafs,omap_out} out, nms_<case>_none = 1 when the level is dropped):
  nan_next_to_max   a NaN beside a finite maximum of 5.0 (MaxPool3d lets NaN through: the maximum is suppressed)
  inf_centre        a +inf response (suppressed by its own window maximum: inf - inf = NaN)
  nan_on_omap       NaN survivors where the octave map is nonzero ((om + NaN).byte() is 0)
  nan_drops_level   two finite maxima, one of them beside a NaN: one positive maximum is left, the level is dropped
"""
import contextlib
import io
import os
import sys
import warnings

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
import ref_harness as R  # noqa: E402

warnings.filterwarnings("ignore")
torch.set_num_threads(8)

HESS_SIGMAS = (1.6, 3.2)
TOPK = 50
SCALE_KS = (54, 57, 58, 60, 61, 63)
OCT1_NAN = (15, 26)          # (y, x) of the NaN in level 1 of octave 1 (32x40)


def base_image(h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return F.avg_pool2d(torch.rand(1, 1, h + 4, w + 4, generator=g) * 255, 5, 1)


def images():
    base, small = base_image(64, 80, 3), base_image(17, 19, 4)
    out = {}

    def put(name, img, y, x, v):
        t = img.clone()
        t[0, 0, y, x] = v
        out[name] = t
    put("nan_mid", base, 31, 40, float("nan"))
    put("nan_edge", base, 0, 45, float("nan"))
    put("nan_corner", base, 63, 79, float("nan"))
    put("pinf", base, 22, 57, float("inf"))
    put("ninf", base, 40, 17, float("-inf"))
    put("small_nan", small, 8, 9, float("nan"))
    out["oct1_nan"] = base.clone()
    for k in SCALE_KS:
        out["scale_%d" % k] = base * (2.0 ** k)
    return out


def detect(det, img, K, patch_oct1=False):
    gen = det.ScalePyrGen
    if patch_oct1:
        def patched(x):
            pyr, sig, pd = type(gen).forward(gen, x)
            pyr[1][1] = pyr[1][1].clone()
            pyr[1][1][0, 0, OCT1_NAN[0], OCT1_NAN[1]] = float("nan")
            return pyr, sig, pd
        gen.forward = patched
    try:
        with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
            r = det.multiScaleDetector(img, K)
    except ValueError:         # torch.cat of an empty list: no level of any octave was accepted
        return [np.zeros(0, np.float32), np.zeros((0, 2, 3), np.float32), np.zeros(0, np.float32), np.zeros(0, np.float32)]
    finally:
        gen.__dict__.pop("forward", None)
    return [t.detach().numpy() for t in r[:4]]


def nms_cases():
    """Response maps [h, w] (h, w = 24, 28) built so each case reaches what its name says."""
    h, w = 24, 28
    g = torch.Generator().manual_seed(7)
    yy, xx = torch.meshgrid(torch.arange(h).float(), torch.arange(w).float(), indexing="ij")

    def blobs(centres, amp):
        m = torch.zeros(h, w)
        for (cy, cx) in centres:
            m += amp * torch.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / 4.0)
        return m
    cases = {}
    spots = [(8, 8), (8, 19), (16, 12), (16, 21)]
    lo, hi = blobs(spots, 1.0), blobs(spots, 1.5)
    cur = blobs(spots, 5.0)
    c = cur.clone(); c[8, 9] = float("nan")                       # the maximum 5.0 at (8, 8) sits beside a NaN
    cases["nan_next_to_max"] = (lo, c, hi, np.zeros((h, w), np.uint8))
    c = cur.clone(); c[16, 12] = float("inf")
    cases["inf_centre"] = (lo, c, hi, np.zeros((h, w), np.uint8))
    c = cur.clone(); c[12, 15] = float("nan")                     # an isolated NaN: a NaN survivor of the NMS
    om = np.zeros((h, w), np.uint8); om[10:14, 13:18] = 3; om[16, 21] = 2
    cases["nan_on_omap"] = (lo, c, hi, om)
    cut = lambda m: torch.where(m > 0.05, m, torch.zeros_like(m))  # noqa: E731   (no plateau of tails within NMS3d's eps)
    c = cut(blobs(spots[:2], 5.0)); c[8, 20] = float("nan")
    cases["nan_drops_level"] = (cut(blobs(spots[:2], 1.0)), c, cut(blobs(spots[:2], 1.5)), np.zeros((h, w), np.uint8))
    noise = (torch.rand(h, w, generator=g) * 1e-3)         # breaks the ties of the flat background (not in nan_drops_level)
    return {k: (a, b, d, om) if k == "nan_drops_level" else (a + noise, b + noise, d + noise, om) for k, (a, b, d, om) in cases.items()}


def main():
    m = R.ref_modules()
    HR = m["HandCraftedModules"].HessianResp()
    det = R.make_detector(None, num_features=TOPK, border=5, mrSize=5.192)
    out = {"hess_sigmas": np.array(HESS_SIGMAS), "topk": np.array(TOPK), "oct1_nan": np.array(OCT1_NAN)}
    for name, img in images().items():
        out["img_" + name] = img.numpy()
        with torch.no_grad():
            for i, s in enumerate(HESS_SIGMAS):
                out["hess_%s_%d" % (name, i)] = HR(img, s).numpy()
        for K in (0, TOPK):
            r = detect(det, img, K, patch_oct1=(name == "oct1_nan"))
            for key, v in zip(("resp", "lafs", "pyr", "lvl"), r):
                out["det%d_%s_%s" % (K, name, key)] = v
    scales = [1.6, 2.0158736798317967, 2.5398416831491195]
    for name, (lo, cur, hi, om) in nms_cases().items():
        h, w = cur.shape
        nms = m["HandCraftedModules"].NMS3dAndComposeA(w=w, h=h, border=5, mrSize=5.192)
        t = lambda a: a.view(1, 1, h, w).float()  # noqa: E731
        with torch.no_grad():
            r, A, om_out = nms(t(lo), t(cur), t(hi), num_features=0, octaveMap=torch.from_numpy(om).view(1, 1, h, w), scales=scales)
        for key, v in (("low", lo), ("cur", cur), ("high", hi)):
            out["nms_%s_%s" % (name, key)] = v.numpy()
        out["nms_%s_omap" % name] = om
        out["nms_%s_none" % name] = np.array(int(r is None))
        if r is not None:
            out["nms_%s_resp" % name] = r.numpy()
            out["nms_%s_lafs" % name] = A.numpy()
            out["nms_%s_omap_out" % name] = om_out.numpy().reshape(h, w)
    out["nms_scales"] = np.array(scales)
    path = os.path.join(HERE, "nonfinite.npz")
    np.savez_compressed(path, **out)
    print("nonfinite.npz %.1f KB, %d arrays" % (os.path.getsize(path) / 1024.0, len(out)))


if __name__ == "__main__":
    main()
