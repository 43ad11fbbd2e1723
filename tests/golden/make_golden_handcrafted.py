"""Generates tests/golden/handcrafted_edges.npz by running the UNMODIFIED reference's OrientationDetector, AffineShapeEstimator
(HandCraftedModules.py) and SIFTNet (pytorch_sift.py) on CPU, through the same harness as make_golden.py (oracle/ref_harness.py).
Re-run only when the reference changes:

    python tests/golden/make_golden_handcrafted.py

For PS in 3, 5, 15, 19, 32, 41 (the estimators) and 16, 32, 41, 65 (SIFT):
  {hc,sift}_patches_PS   [n,PS,PS] fp32: edge_patches(PS) below, then N_RANDOM seeded patches of integer grey levels
  ori_gk_PS, aff_gk_PS   the modules' Gaussian windows (OrientationDetector's is 10x the kernel, rounded to fp32 as torch does)
  ori_angle_PS           OrientationDetector(patch_size=PS) -> angle [n]
  aff_A_PS               AffineShapeEstimator(patch_size=PS) -> rectified A [n,2,2]
  sift_desc_PS           SIFTNet(patch_size=PS) -> [n,128]
  edge_names             the names of the edge patches, in order
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
import ref_harness as R  # noqa: E402
from handcrafted_restated import EDGE_NAMES, edge_patches  # noqa: E402

warnings.filterwarnings("ignore")
HC_PS = (3, 5, 15, 19, 32, 41)
SIFT_PS = (16, 32, 41, 65)
N_RANDOM = 6


def patches(PS, seed):
    g = torch.Generator().manual_seed(seed)
    rnd = torch.floor(torch.rand(N_RANDOM, PS, PS, generator=g) * 256.0).numpy()
    return np.concatenate([edge_patches(PS), rnd]).astype(np.float32)


def main():
    m = R.ref_modules()
    HC = m["HandCraftedModules"]
    PSIFT = importlib.import_module("pytorch_sift")
    out = {"edge_names": np.array(EDGE_NAMES)}
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
        for PS in HC_PS:
            P = patches(PS, 100 + PS)
            x = torch.from_numpy(P).view(-1, 1, PS, PS)
            ori, aff = HC.OrientationDetector(patch_size=PS), HC.AffineShapeEstimator(patch_size=PS)
            out["hc_patches_%d" % PS] = P
            out["ori_angle_%d" % PS] = ori(x).numpy()
            out["aff_A_%d" % PS] = aff(x).numpy()
            out["ori_gk_%d" % PS], out["aff_gk_%d" % PS] = ori.gk.numpy(), aff.gk.numpy()
        for PS in SIFT_PS:
            P = patches(PS, 200 + PS)
            sift = PSIFT.SIFTNet(patch_size=PS)
            out["sift_patches_%d" % PS] = P
            out["sift_desc_%d" % PS] = sift(torch.from_numpy(P).view(-1, 1, PS, PS)).numpy()
    path = os.path.join(HERE, "handcrafted_edges.npz")
    np.savez_compressed(path, **out)
    print("handcrafted_edges.npz %.1f KB" % (os.path.getsize(path) / 1024.0))


if __name__ == "__main__":
    main()
