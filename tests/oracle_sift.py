"""CPU restatement of the SIFT descriptor (SIFTNet, pytorch_sift.py:30-94) with 8 angle bins x 4 x 4 spatial bins, written from the
algorithm and pinned to the unmodified reference by tests/golden/sift.npz (tests/test_sift_cpu.py).  Test infrastructure only, as
oracle/affnet_oracle.py, whose pyramid level choice and sampler `describe_sift` reuses.  Also defines the constructed patches of the
golden set, so that tests/golden/make_golden_sift.py and the tests build the same patches without storing them."""
import math

import numpy as np
import torch
import torch.nn.functional as F

import affnet_oracle as O

def sift_geometry(PS):
    """Pooling stride s = round(2 floor(PS/2) / 5) and kernel size k = 2 s - 1 of a PS x PS patch."""
    s = int(round(2.0 * (PS // 2) / 5.0))
    return 2 * s - 1, s


def sift_windows(PS):
    """(gk [PS,PS], pk [k,k]) as fp32: a circular Gaussian centred at PS/2 (a half-integer for odd PS) with sigma^2 = 0.9 r^2, r = PS/2,
    zero from radius r on and not normalised; and the separable tent kernel whose 1-D profile rises in steps of 1/floor(k/2) from half
    a step to 1 and back."""
    half = PS / 2.0
    d = np.arange(PS, dtype=np.float64) - half
    disq = d.reshape(-1, 1) ** 2 + d.reshape(1, -1) ** 2
    gk = np.where(disq < half * half, np.exp(-disq / (0.9 * half * half)), 0.0)
    k, _ = sift_geometry(PS)
    step = 1.0 / float(k // 2)
    ramp = np.arange(step / 2.0, 1.0, step)
    prof = np.concatenate([ramp, [1.0], ramp[::-1]])
    return torch.from_numpy(gk.astype(np.float32)), torch.from_numpy(np.maximum(np.outer(prof, prof), 0.0).astype(np.float32))


def sift_describe(patches, clipval=0.2):
    """SIFT of [n,1,PS,PS] patches -> [n,128] in [angle bin][cell y][cell x] order: central-difference gradients with replicate borders,
    magnitude sqrt(gx^2 + gy^2 + 1e-10) times the Gaussian window, angle atan2(gy, gx + 1e-8) mapped to o = (angle + 2 pi) / (2 pi) * 8
    and split linearly between bins floor(o) % 8 and (floor(o) + 1) % 8, per-bin tent pooling (k x k, stride s, no padding), then
    L2 normalisation (sqrt(|sum x^2| + 1e-10)), clamp(0, clipval) and L2 normalisation again."""
    x = patches.float()
    n, PS = x.size(0), x.size(2)
    gk, pk = sift_windows(PS)
    k, s = sift_geometry(PS)
    xp = F.pad(x, (1, 1, 0, 0), "replicate")
    gx = xp[:, :, :, 2:] - xp[:, :, :, :-2]
    yp = F.pad(x, (0, 0, 1, 1), "replicate")
    gy = yp[:, :, 2:, :] - yp[:, :, :-2, :]
    mag = torch.sqrt(gx * gx + gy * gy + 1e-10) * gk
    o = (torch.atan2(gy, gx + 1e-8) + 2.0 * math.pi) / (2.0 * math.pi) * 8.0
    b0 = torch.floor(o)
    frac = o - b0
    b0 = b0 % 8
    b1 = (b0 + 1) % 8
    maps = torch.cat([(b0 == i).float() * ((1.0 - frac) * mag) + (b1 == i).float() * (frac * mag) for i in range(8)], dim=1)
    pooled = F.conv2d(maps.reshape(n * 8, 1, PS, PS), pk.view(1, 1, k, k), stride=s).reshape(n, -1)

    def l2(v):
        return v / torch.sqrt(torch.abs((v * v).sum(dim=1)) + 1e-10).unsqueeze(1)

    return l2(torch.clamp(l2(pooled), 0.0, float(clipval)))


def describe_sift(dLAFs, state, PS=32, clipval=0.2):
    """extract_patches_from_pyr (SparseImgRepresenter.py:181-188) at patch size PS + the SIFT descriptor; `state` of O.detect."""
    pyr = state["pyr"]
    o, l = O.pyramid_level_for_lafs(dLAFs, state["sigmas"], state["pix_dists"], PS)
    nl = O.normalize_lafs(dLAFs, pyr[0][0].size(3), pyr[0][0].size(2))
    patches = O.extract_patches_from_pyramid(pyr, o, l, nl, PS)
    return sift_describe(patches, clipval), patches, (o, l)


def constructed_patches(PS):
    """[9,1,PS,PS]: zero, constant, horizontal / vertical ramps of both signs (gradient angles on bin boundaries; the falling horizontal
    ramp has gy = 0, gx < 0 everywhere: the +-pi cut), a diagonal ramp (45 degrees), a checkerboard, and a ramp with a small
    deterministic ripple, where the clip at 0.2 binds on most of the 16 cells of the dominant bin."""
    i = torch.arange(PS, dtype=torch.float32).view(PS, 1).expand(PS, PS)
    j = torch.arange(PS, dtype=torch.float32).view(1, PS).expand(PS, PS)
    ripple = ((7 * i + 13 * j) % 11) * 0.02
    P = [torch.zeros(PS, PS), torch.full((PS, PS), 97.0), 3.0 * j, 200.0 - 3.0 * j, 3.0 * i, 200.0 - 3.0 * i, 2.0 * i + 2.0 * j,
         255.0 * ((i + j) % 2), 2.0 * j + ripple]
    return torch.stack(P).view(-1, 1, PS, PS).contiguous()


def golden_patches(z, name, PS):
    """The patches of tests/golden/sift.npz (`z`) that the reference described: integer grey levels (uint8), graf descriptor patches
    (float16, exactly the reference's input) or the constructed set."""
    if name == "random":
        return torch.from_numpy(z["random_u8_%d" % PS]).float()
    if name == "graf":
        return torch.from_numpy(z["graf_f16_%d" % PS]).float()
    return constructed_patches(PS)
