"""HardNet with the reference's interface (HardNet.py:61-101), executed by the sm_90a CUDA library:
[n,1,32,32] -> L2-normalised [n,128].  `features.*` names match HardNet++.pth."""
import torch
import torch.nn as nn

from . import _lib as L
from ._nets import HARD_CFG, _NativeNet, make_features


class HardNet(_NativeNet):
    KIND = L.NET_HARDNET

    def __init__(self):
        super().__init__()
        self.features = make_features(HARD_CFG, [nn.Dropout(0.1), nn.Conv2d(128, 128, kernel_size=8, bias=False),
                                                 nn.BatchNorm2d(128, affine=False)])

    def forward(self, input):
        x = self._check_input(input)
        n = x.size(0)
        out = torch.empty(n, 128, dtype=torch.float32, device=x.device)
        if n == 0:
            return out
        ws, nbytes = self._workspace(n, x.device)
        L.check(L.lib().ag_hardnet_forward(self.handle(), L.ptr(x), n, None, 0, L.ptr(out), L.ptr(ws), nbytes, L.stream_ptr()))
        return out
