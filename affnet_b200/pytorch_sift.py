"""pytorch_sift.py counterpart: SIFTNet (:30-94), the hand-crafted SIFT descriptor, on the GPU (ag_sift_describe).  Used as the reference's
scripts use it, in place of HardNet: `desc = SIFTNet(patch_size=32)` on `det.extract_patches_from_pyr(LAFs, PS=32)`, or in the HardNet
position of DetectDescribePipeline."""
import ctypes as C

import numpy as np
import torch
import torch.nn as nn

from . import _lib as L


class SIFTNet(nn.Module):
    """SIFTNet(patch_size=65, num_ang_bins=8, num_spatial_bins=4, clipval=0.2): forward([n,1,PS,PS]) -> [n,128].  Only the reference's
    8 angle bins x 4 x 4 spatial bins are supported; patch sizes 16..65 whose pooling grid comes out 4 x 4."""

    def __init__(self, patch_size=65, num_ang_bins=8, num_spatial_bins=4, clipval=0.2):
        super().__init__()
        if num_ang_bins != 8 or num_spatial_bins != 4:
            raise L.AffnetB200Error("SIFTNet: only num_ang_bins=8 and num_spatial_bins=4 are supported, got %r and %r"
                                    % (num_ang_bins, num_spatial_bins))
        self.patch_size, self.PS = int(patch_size), int(patch_size)
        self.num_ang_bins, self.num_spatial_bins = num_ang_bins, num_spatial_bins
        self.clipval = float(clipval)
        if not (np.isfinite(self.clipval) and self.clipval > 0.0):
            raise L.AffnetB200Error("SIFTNet: clipval must be finite and positive, got %r" % clipval)
        PS = self.PS
        gk = np.zeros(PS * PS, np.float32)
        pk = np.zeros(25 * 25, np.float32)
        k, s = C.c_int(), C.c_int()
        L.check(L.lib().ag_sift_windows(PS, gk.ctypes.data_as(C.c_void_p), pk.ctypes.data_as(C.c_void_p), C.byref(k), C.byref(s)))
        self.bin_weight_kernel_size, self.bin_weight_stride = k.value, s.value
        self.gk = torch.from_numpy(gk.reshape(PS, PS))
        self.pk = torch.from_numpy(pk[:k.value * k.value].reshape(k.value, k.value).copy())

    def forward(self, x):
        x = L.f32c(x, "patches")
        if x.dim() != 4 or x.size(1) != 1 or x.size(2) != self.PS or x.size(3) != self.PS:
            raise L.AffnetB200Error("expected patches of shape [n,1,%d,%d]" % (self.PS, self.PS))
        n = x.size(0)
        out = torch.empty(n, 128, dtype=torch.float32, device=x.device)
        if n:
            L.check(L.lib().ag_sift_describe(L.ptr(x), n, self.PS, self.clipval, L.ptr(out), L.stream_ptr()))
        return out
