#!/usr/bin/env python
"""Counterpart of the reference's examples/hesaffnet/hesaffnet.py on the H100-native path:

    python examples/hesaffnet.py img.png out.txt 2000 [--weights tests/golden/weights.npz | --affnet pretrained/AffNet.pth] [--th 28.41]

writes the Oxford-affine ellipse file (`1.0`, N, then `x y a b c` rows, %10.10f) exactly like hesaffnet.py:56-60.
--th runs the reference's threshold mode (hesaffnet.py:25-26 sets th = -1; 28.41 is its HessianAffine default): every keypoint above
the threshold, nfeats is then ignored.  Without --th the top nfeats keypoints are kept.
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from affnet_b200.architectures import AffNetFast  # noqa: E402
from affnet_b200.LAF import LAFs2ell  # noqa: E402
from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor  # noqa: E402
from affnet_b200.Utils import line_prepender  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("image"); ap.add_argument("output"); ap.add_argument("nfeats", type=int)
    ap.add_argument("--affnet", default=None, help="AffNet.pth of the reference (state_dict under 'state_dict')")
    ap.add_argument("--weights", default=os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "weights.npz"))
    ap.add_argument("--th", type=float, default=None, help="Hessian threshold: keep every keypoint above it (the reference's -1 or 28.41)")
    args = ap.parse_args()
    from PIL import Image
    img = np.mean(np.array(Image.open(args.image).convert("RGB")), axis=2)                      # hesaffnet.py:35-36
    x = torch.from_numpy(img.astype(np.float32)).view(1, 1, img.shape[0], img.shape[1]).cuda()
    net = AffNetFast(PS=32)
    if args.affnet:
        net.load_state_dict(torch.load(args.affnet, map_location="cpu")["state_dict"])
    else:
        z = np.load(args.weights)
        net.load_state_dict({k.split("/", 1)[1]: torch.from_numpy(z[k]) for k in z.files if k.startswith("affnet/")})
    net = net.eval().cuda()
    HA = ScaleSpaceAffinePatchExtractor(mrSize=5.192, num_features=args.nfeats, border=5, num_Baum_iters=1, th=args.th, AffNet=net)
    with torch.no_grad():
        LAFs, resp = HA(x)
    ells = LAFs2ell(LAFs.cpu().numpy())
    np.savetxt(args.output, ells, delimiter=" ", fmt="%10.10f")
    line_prepender(args.output, str(len(ells)))
    line_prepender(args.output, "1.0")
    print("%d regions -> %s" % (len(ells), args.output))


if __name__ == "__main__":
    main()
