"""LAF helpers with the reference's names (LAF.py): the affine sampler, (de)normalisation, level routing and the
Oxford-ellipse conversions in both directions."""
import ctypes as C

import numpy as np
import torch

from . import _lib as L


def extract_patches(img, LAFs, PS=32, bs=32):
    """LAF.py:364-372.  img [1|n,C,h,w] CUDA float32, LAFs [n,2,3] normalised -> [n,C,PS,PS].
    `bs` (a memory-chunking knob in the reference) is accepted and ignored."""
    img = L.f32c(img, "img")
    LAFs = L.f32c(LAFs, "LAFs")
    n = LAFs.size(0)
    Cc, h, w = img.size(1), img.size(2), img.size(3)
    per_patch = 1 if (img.size(0) == n and n != 1) else 0
    if not per_patch and img.size(0) != 1:
        raise L.AffnetB200Error("img batch must be 1 or equal to the number of LAFs")
    out = torch.empty(n, Cc, PS, PS, dtype=torch.float32, device=img.device)
    step = 65535
    for s in range(0, n, step):
        e = min(n, s + step)
        src = img[s:e] if per_patch else img
        L.check(L.lib().ag_extract_patches(L.ptr(src), Cc, h, w, per_patch, L.ptr(LAFs[s:e]), e - s, PS, L.ptr(out[s:e]), L.stream_ptr()))
    return out


def _scale(LAFs, ac, xc, yc):
    LAFs = L.f32c(LAFs, "LAFs")
    out = torch.empty_like(LAFs)
    if LAFs.size(0) == 0:
        return out
    L.check(L.lib().ag_lafs_scale(L.ptr(LAFs), L.ptr(out), LAFs.size(0), ac, xc, yc, L.stream_ptr()))
    return out


def denormalizeLAFs(LAFs, w, h):
    """LAF.py:407-417."""
    w, h = float(w), float(h)
    return _scale(LAFs, min(h, w), w, h)


def normalizeLAFs(LAFs, w, h):
    """LAF.py:419-429 (coefficients rounded to float32 exactly as the reference's coef tensor)."""
    w, h = float(w), float(h)
    ms = np.float32(min(h, w))
    return _scale(LAFs, float(np.float32(1.0) / ms), float(np.float32(1.0 / w)), float(np.float32(1.0 / h)))


def get_pyramid_and_level_index_for_LAFs(dLAFs, plan, PS):
    """LAF.py:453-472 (float64 argmin on device instead of scipy cdist on the host).  `plan` is the pyramid plan
    of the detector (carries sigmas and pixel distances).  Returns int32 (octave, level) tensors."""
    dLAFs = L.f32c(dLAFs, "dLAFs")
    n = dLAFs.size(0)
    o = torch.empty(n, dtype=torch.int32, device=dLAFs.device)
    l = torch.empty(n, dtype=torch.int32, device=dLAFs.device)
    if n == 0:
        return o, l
    L.check(L.lib().ag_pyramid_level_for_lafs(C.byref(plan), L.ptr(dLAFs), n, PS, L.ptr(o), L.ptr(l), L.stream_ptr()))
    return o, l


def get_LAFs_scales(LAFs):
    return torch.sqrt(torch.abs(LAFs[:, 0, 0] * LAFs[:, 1, 1] - LAFs[:, 0, 1] * LAFs[:, 1, 0]) + 1e-12)


def LAFs2ell(in_LAFs):
    """LAF.py:225-240: [n,2,3] numpy LAFs -> [x y a b c] ellipse rows (host-side output format).  As in the reference the SVD runs
    in the dtype of the input (float32 for `LAFs.cpu().numpy()`, hesaffnet.py:56) and the rows are returned as float64."""
    LAFs = np.asarray(in_LAFs)
    if not np.issubdtype(LAFs.dtype, np.floating):
        LAFs = LAFs.astype(np.float64)
    LAFs = LAFs.reshape(-1, 2, 3)
    ell = np.zeros((len(LAFs), 5))
    for i in range(len(LAFs)):
        A = LAFs[i, :, :2]
        scale = np.sqrt(A[0, 0] * A[1, 1] - A[0, 1] * A[1, 0] + 1e-10)
        u, W, _ = np.linalg.svd(A / scale, full_matrices=True)
        W = 1.0 / (W * W * scale * scale)
        M = np.matmul(np.matmul(u, np.diag(W)), u.transpose())
        ell[i] = [LAFs[i, 0, 2], LAFs[i, 1, 2], M[0, 0], M[0, 1], M[1, 1]]
    return ell


def LAFs2ellT(LAFs):
    """LAF.py:35-51 on the device (`ag_lafs_to_ell`): [n,2,3] pixel LAFs -> [n,5] rows (x, y, a, b, c), the Oxford-affine
    format hesaffBaum.py:46-48 writes."""
    if not LAFs.is_cuda:
        raise L.AffnetB200Error("LAFs2ellT: CUDA tensor expected (there is no CPU path)")
    LAFs = LAFs.contiguous().float()
    n = LAFs.size(0)
    ell = torch.empty(n, 5, device=LAFs.device)
    if n:
        L.check(L.lib().ag_lafs_to_ell(L.ptr(LAFs), n, L.ptr(ell), L.stream_ptr()))
    return ell


def ells2LAFsT(ells):
    """LAF.py:76-89 on the device (`ag_ells_to_lafs`): [n,5] Oxford-affine rows (x, y, a, b, c) -> [n,2,3] upright pixel LAFs, the
    reference's fp32 arithmetic bit for bit (NaN for an ellipse that is not positive definite, as there)."""
    if not ells.is_cuda:
        raise L.AffnetB200Error("ells2LAFsT: CUDA tensor expected (there is no CPU path)")
    ells = ells.contiguous().float().view(-1, 5)
    n = ells.size(0)
    lafs = torch.empty(n, 2, 3, device=ells.device)
    if n:
        L.check(L.lib().ag_ells_to_lafs(L.ptr(ells), n, L.ptr(lafs), L.stream_ptr()))
    return lafs


def save_ells(fname, ells):
    """The reference's text output (hesaffBaum.py:48): one `x y a b c` row per keypoint, %10.10f."""
    np.savetxt(fname, ells.detach().cpu().numpy() if isinstance(ells, torch.Tensor) else np.asarray(ells), delimiter=" ", fmt="%10.10f")
