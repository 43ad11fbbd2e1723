"""Generates tests/golden/threshold.npz by running the UNMODIFIED reference (/root/reference, ducha-aiki/affnet) on CPU in its threshold
mode, as its command-line detector examples/hesaffnet/hesaffnet.py builds it:

    ScaleSpaceAffinePatchExtractor(mrSize=5.192, num_features=nfeats, border=5, num_Baum_iters=1, th=th, AffNet=AffNetFast)

with no orientation (hesaffnet.py calls HA(x) with do_ori=False).  With th set, num_features is ignored (SparseImgRepresenter.py:33-37):
every keypoint above th is kept, and every survivor of the shape filter.

    python tests/golden/make_golden_threshold.py

Outputs (threshold.npz, compressed):
  th28_resp, th28_dLAFs   test-graf/img1.png (800x640), th = 28.41 (hesaffnet.py's "default threshold for HessianAffine")
  thm1_resp, thm1_dLAFs   the 256x320 graf crop of graf_crop.npz, th = -1 (the value hesaffnet.py runs)
"""
import contextlib
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


def gray_of(rgb):
    return torch.from_numpy(np.mean(rgb, axis=2).astype(np.float32)).view(1, 1, rgb.shape[0], rgb.shape[1])


def run(aff, img, th):
    det = R.make_detector(aff, num_features=2000, border=5, mrSize=5.192, th=th)
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
        LAFs, resp = det(img, do_ori=False)
    return resp.detach().numpy(), LAFs.detach().numpy()


def main():
    aff, _, _ = R.load_nets()
    full = gray_of(np.load(os.path.join(HERE, "graf_full.npz"))["rgb"])
    crop = gray_of(np.load(os.path.join(HERE, "graf_crop.npz"))["rgb"])
    out = {}
    out["th28_resp"], out["th28_dLAFs"] = run(aff, full, 28.41)
    out["thm1_resp"], out["thm1_dLAFs"] = run(aff, crop, -1)
    path = os.path.join(HERE, "threshold.npz")
    np.savez_compressed(path, **out)
    print("threshold.npz %.1f KB: %d keypoints at th 28.41, %d at th -1" % (os.path.getsize(path) / 1024.0, len(out["th28_resp"]),
                                                                            len(out["thm1_resp"])))


if __name__ == "__main__":
    main()
