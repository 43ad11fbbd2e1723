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
