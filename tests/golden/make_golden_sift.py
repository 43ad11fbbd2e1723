"""Generates tests/golden/sift.npz by running the UNMODIFIED reference's SIFTNet (pytorch_sift.py) on CPU, through the same harness as
make_golden.py (oracle/ref_harness.py).  Re-run only when the reference changes:

    python tests/golden/make_golden_sift.py

For PS in 16, 32, 41, 65:
  gk_PS, pk_PS, k_PS, stride_PS      SIFTNet(PS)'s Gaussian window, pooling kernel, kernel size and stride
  random_u8_PS                       4 seeded random patches of integer grey levels (stored exactly as uint8)
  graf_f16_PS                        4 descriptor patches of the graf crop (extract_patches_from_pyr(dLAFs, PS), AffNet + histogram
                                     orientation, K = 300), rounded to float16 BEFORE the reference describes them, so the stored patches
                                     are exactly its input while the file stays small
  {random,graf,constructed}_desc_PS  the reference's descriptors of those patches and of tests/oracle_sift.py::constructed_patches(PS)
And graf img1 <-> img6 with SIFTNet(32) in place of HardNet (AffNet, K = 3000, SNN 0.8, 6 px; train_AffNet_test_on_graffity.py:262-300),
with hand-crafted orientation (hcori_*) and without (noori_*): keypoint counts, tentative and true matches.
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
sys.path.insert(0, os.path.join(HERE, ".."))
import oracle_sift as OS  # noqa: E402
import ref_harness as R  # noqa: E402

warnings.filterwarnings("ignore")
torch.set_num_threads(8)
SIFT_PS = (16, 32, 41, 65)
N_RANDOM, N_GRAF = 4, 4


def quiet():
    return contextlib.redirect_stdout(io.StringIO())


def rgb_of(path):
    from PIL import Image
    return np.array(Image.open(path).convert("RGB"))


def gray_of(rgb):
    return torch.from_numpy(np.mean(rgb, axis=2).astype(np.float32)).view(1, 1, rgb.shape[0], rgb.shape[1])


def main():
    R.ref_modules()
    PSIFT = importlib.import_module("pytorch_sift")
    RS, LS = importlib.import_module("ReprojectionStuff"), importlib.import_module("Losses")
    aff, _, _ = R.load_nets()
    out = {}
    crop = np.load(os.path.join(HERE, "graf_crop.npz"))["rgb"]
    det = R.make_detector(aff, None, num_features=300)
    with torch.no_grad(), quiet():
        dL, _ = det(gray_of(crop), do_ori=True)
    g = torch.Generator().manual_seed(29)
    for PS in SIFT_PS:
        sift = PSIFT.SIFTNet(patch_size=PS)
        out["gk_%d" % PS] = sift.gk
        out["pk_%d" % PS] = sift.pk[0].weight.data[0, 0]
        out["k_%d" % PS], out["stride_%d" % PS] = sift.bin_weight_kernel_size, sift.bin_weight_stride
        rnd = torch.floor(torch.rand(N_RANDOM, 1, PS, PS, generator=g) * 256.0)
        with torch.no_grad(), quiet():
            graf = det.extract_patches_from_pyr(dL, PS=PS)[:N_GRAF].half()
        out["random_u8_%d" % PS], out["graf_f16_%d" % PS] = rnd.to(torch.uint8), graf
        with torch.no_grad():
            out["random_desc_%d" % PS] = sift(rnd)
            out["graf_desc_%d" % PS] = sift(graf.float().contiguous())
            out["constructed_desc_%d" % PS] = sift(OS.constructed_patches(PS))
    rgb1, rgb6 = rgb_of(R.REF + "/test-graf/img1.png"), rgb_of(R.REF + "/test-graf/img6.png")
    H = np.loadtxt(R.REF + "/test-graf/H1to6p")
    out.update(K=3000, snn=0.8, px=6.0)
    sift = PSIFT.SIFTNet(patch_size=32)
    for mode in ("hcori", "noori"):
        det = R.make_detector(aff, None, num_features=3000)
        L1, _, _, d1 = R.run_full(det, sift, gray_of(rgb1), mode != "noori")
        L2, _, _, d2 = R.run_full(det, sift, gray_of(rgb6), mode != "noori")
        with torch.no_grad():                                       # train_AffNet_test_on_graffity.py:289-300
            dm = LS.distance_matrix_vector(d1, d2)
            mn, i2 = torch.min(dm, 1)
            dm[:, i2] = 100000
            sec, _ = torch.min(dm, 1)
            mask = (mn / (sec + 1e-8)) <= 0.8
            t1, t2 = torch.arange(0, i2.size(0))[mask].long(), i2[mask].long()
            _, pi1, _ = RS.get_GT_correspondence_indexes(L1[t1], L2[t2], torch.from_numpy(H).float(), dist_threshold=6)
        out.update({mode + "_n1": L1.size(0), mode + "_n2": L2.size(0), mode + "_tent": t1.numel(), mode + "_true": pi1.numel()})
        print(mode, L1.size(0), L2.size(0), t1.numel(), "tentatives", pi1.numel(), "true")
    path = os.path.join(HERE, "sift.npz")
    np.savez_compressed(path, **{k: (v.detach().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in out.items()})
    print("sift.npz %.1f KB" % (os.path.getsize(path) / 1024.0))


if __name__ == "__main__":
    main()
