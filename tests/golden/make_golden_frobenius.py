"""Generates tests/golden/frobenius.npz by running the UNMODIFIED reference (/root/reference, ducha-aiki/affnet) on CPU, through the same
harness as make_golden.py (oracle/ref_harness.py).  Re-run only when the reference changes:

    python tests/golden/make_golden_frobenius.py

The reference's two Frobenius functions hard-code batch_size = 2 in reproject_to_canonical_Frob_batched, which scrambles the distance
matrix (DESIGN.md, Frobenius quirk 1).  To record the intended matrix, the module attribute is replaced by a wrapper that calls the
original with batch_size = 1 (a shim: no reference source is copied or edited); the raw batch_size = 2 matrices are stored as well.

Outputs (frobenius.npz, compressed):
  H1to6, lafs1, lafs6     graf img1 / img6, the reference detector's pixel LAFs with AffNet and no orientation at K = 3000 (the "noori"
                          run of graf_match.npz, whose tentatives noori_t1 / noori_t2 index these rows)
  set_<case>_{min,i1,i2}  the function on (lafs1, lafs6, H1to6) at dist_threshold = +inf: every row whose minimum is not NaN
  tent_<case>_{min,i1,i2} the same on the tentatives (lafs1[t1], lafs6[t2])
  <mode>_l2in1            return_LAF2_in_1's LAF2_in_1 for the default flags
        cases: fro, fro_skip (get_GT_correspondence_indexes_Fro), fc, fc_skip, fc_up, fc_noinv, fc_noinv_skip
        (get_GT_correspondence_indexes_Fro_and_center: defaults, skip_center_in_Fro, do_up_is_up, inv_to_eye = False)
  tent_D1, tent_D2        reproject_to_canonical_Frob_batched on the tentatives with batch_size 1 and 2
  rnd_l1, rnd_l2, rnd_H   a small random case (7 x 9) with a NaN column (2) and an infinite one (5) in side 2
  rnd_D1, rnd_D2          its matrices with batch_size 1 and 2; rnd_<case>_{min,i1,i2} for fro and fc
  err_scale0, err_singular  the exception the reference raises for scale_diff_coef = 0, and for a singular row of LAFs1
"""
import contextlib
import importlib
import io
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
import ref_harness as R  # noqa: E402

warnings.filterwarnings("ignore")
torch.set_num_threads(8)
INF = float("inf")


def gray_of(rgb):
    return torch.from_numpy(np.mean(rgb, axis=2).astype(np.float32)).view(1, 1, rgb.shape[0], rgb.shape[1])


def cases(RS):
    fro, fc = RS.get_GT_correspondence_indexes_Fro, RS.get_GT_correspondence_indexes_Fro_and_center
    return {"fro": (fro, {}), "fro_skip": (fro, dict(skip_center_in_Fro=True)), "fc": (fc, {}), "fc_skip": (fc, dict(skip_center_in_Fro=True)),
            "fc_up": (fc, dict(do_up_is_up=True)), "fc_noinv": (fc, dict(inv_to_eye=False)),
            "fc_noinv_skip": (fc, dict(inv_to_eye=False, skip_center_in_Fro=True))}


def run(out, tag, fn, kw, L1, L2, H):
    mn, i1, i2 = fn(L1, L2, H, dist_threshold=INF, **kw)[:3]
    out[tag + "_min"], out[tag + "_i1"], out[tag + "_i2"] = mn, i1.long(), i2.long()


def main():
    R.ref_modules()
    RS = importlib.import_module("ReprojectionStuff")
    LAF = importlib.import_module("LAF")
    orig = RS.reproject_to_canonical_Frob_batched

    def batch1(LHF1_inv, LHF2, batch_size=2, skip_center=False):
        return orig(LHF1_inv, LHF2, batch_size=1, skip_center=skip_center)

    def raw(L1, L2, H, bs):
        LHF2 = RS.reprojectLAFs(L2, torch.inverse(H), True)
        return orig(RS.inverseLHFs(LAF.LAFs_to_H_frames(L1)), LHF2, batch_size=bs)

    from PIL import Image
    rgb1 = np.array(Image.open(R.REF + "/test-graf/img1.png").convert("RGB"))
    rgb6 = np.array(Image.open(R.REF + "/test-graf/img6.png").convert("RGB"))
    m = np.load(os.path.join(HERE, "graf_match.npz"))
    H = torch.from_numpy(m["H1to6"]).float()
    aff, _, _ = R.load_nets()
    det = R.make_detector(aff, None, num_features=3000)
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
        L1, _ = det(gray_of(rgb1), do_ori=False)
        L6, _ = det(gray_of(rgb6), do_ori=False)
    assert (L1.size(0), L6.size(0)) == (int(m["noori_n1"]), int(m["noori_n2"])), (L1.size(0), L6.size(0))
    t1, t2 = torch.from_numpy(m["noori_t1"]), torch.from_numpy(m["noori_t2"])
    out = dict(H1to6=H, lafs1=L1, lafs6=L6)

    g = torch.Generator().manual_seed(7)
    rl1 = torch.randn(7, 2, 3, generator=g) * torch.tensor([[3.0, 1.0, 20.0], [1.0, 3.0, 20.0]]) + torch.tensor([[6.0, 0, 50], [0, 6.0, 50]])
    rl2 = rl1[torch.tensor([0, 1, 2, 3, 4, 5, 6, 0, 3])].clone()
    rl2[:, :, 2] += torch.randn(9, 2, generator=g) * 1.5
    rl2[:, :, :2] *= 1.0 + 0.2 * torch.randn(9, 1, 1, generator=g)
    rl2[2, 0, 1] = float("nan")
    rl2[5, 1, 2] = float("inf")
    rH = torch.eye(3) + 0.01 * torch.randn(3, 3, generator=g)
    rH[2, 2] = 1.0
    out.update(rnd_l1=rl1, rnd_l2=rl2, rnd_H=rH)

    with torch.no_grad():
        out["tent_D1"], out["tent_D2"] = raw(L1[t1], L6[t2], H, 1), raw(L1[t1], L6[t2], H, 2)
        out["rnd_D1"], out["rnd_D2"] = raw(rl1, rl2, rH, 1), raw(rl1, rl2, rH, 2)
        RS.reproject_to_canonical_Frob_batched = batch1
        try:
            for tag, (fn, kw) in cases(RS).items():
                run(out, "set_" + tag, fn, kw, L1, L6, H)
                run(out, "tent_" + tag, fn, kw, L1[t1], L6[t2], H)
                if tag in ("fro", "fc"):
                    run(out, "rnd_" + tag, fn, kw, rl1, rl2, rH)
                print(tag, "set rows", out["set_" + tag + "_i1"].numel(), "tentative rows", out["tent_" + tag + "_i1"].numel())
            fc = RS.get_GT_correspondence_indexes_Fro_and_center
            out["set_l2in1"] = fc(L1, L6, H, return_LAF2_in_1=True)[3]
            out["tent_l2in1"] = fc(L1[t1], L6[t2], H, return_LAF2_in_1=True)[3]
            for key, call in (("err_scale0", lambda: fc(rl1, rl2, rH, scale_diff_coef=0.0)),
                              ("err_singular", lambda: RS.get_GT_correspondence_indexes_Fro(
                                  torch.cat([rl1[:3], torch.tensor([[[1.0, 2.0, 5.0], [2.0, 4.0, 5.0]]])]), rl2, rH))):
                try:
                    call()
                    out[key] = ""
                except Exception as e:                                  # noqa: BLE001 (the exception is the recorded result)
                    out[key] = type(e).__name__
                print(key, repr(out[key]))
        finally:
            RS.reproject_to_canonical_Frob_batched = orig
    path = os.path.join(HERE, "frobenius.npz")
    np.savez_compressed(path, **{k: (v.detach().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in out.items()})
    print("frobenius.npz %.1f KB" % (os.path.getsize(path) / 1024.0))


if __name__ == "__main__":
    main()
