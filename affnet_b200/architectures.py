"""AffNetFast / OriNetFast with the reference's interface (architectures.py:204-252, 33-82), executed by the
sm_90a CUDA library.  Same constructor arguments, same `features.*` parameter names (checkpoints load
unchanged), same outputs: AffNetFast -> rectified [n,2,2]; OriNetFast -> rotation [n,2,2] or angle [n]."""
import torch
import torch.nn as nn

from . import _lib as L
from ._nets import AFF_CFG, _NativeNet, make_features


class AffNetFast(_NativeNet):
    KIND = L.NET_AFFNET

    def __init__(self, PS=32):
        super().__init__()
        if PS != 32:
            raise L.AffnetB200Error("AffNetFast kernels are built for PS=32 (the shipped checkpoint)")
        self.features = make_features(AFF_CFG, [nn.Dropout(0.25), nn.Conv2d(64, 3, kernel_size=8, stride=1, padding=0, bias=True),
                                                nn.Tanh(), nn.AdaptiveAvgPool2d(1)])
        self.PS = PS
        self.halfPS = int(PS / 2)

    def forward(self, input, return_A_matrix=False):
        x = self._check_input(input)
        n = x.size(0)
        out = torch.empty(n, 2, 2, dtype=torch.float32, device=x.device)
        if n == 0:
            return out
        ws, nbytes = self._workspace(n, x.device)
        L.check(L.lib().ag_affnet_forward(self.handle(), L.ptr(x), n, None, 0, L.ptr(out), L.ptr(ws), nbytes, L.stream_ptr()))
        return out

    def forward_raw(self, input):
        """The TorchScript export's contract (convertJIT/AffNetJIT.pt): xy + [1, 0, 1] -> [n,3], before rectification."""
        x = self._check_input(input)
        n = x.size(0)
        out = torch.empty(n, 3, dtype=torch.float32, device=x.device)
        if n:
            ws, nbytes = self._workspace(n, x.device)
            L.check(L.lib().ag_affnet_forward_raw(self.handle(), L.ptr(x), n, L.ptr(out), L.ptr(ws), nbytes, L.stream_ptr()))
        return out


class OriNetFast(_NativeNet):
    KIND = L.NET_ORINET

    def __init__(self, PS=16):
        super().__init__()
        # the reference's head kernel is int(PS/4) with padding 1; the shipped OriNet.pth is PS=32 (8x8 head) and every caller of the
        # reference passes PS=32 (train_AffNet_test_on_graffity.py:74, examples/hesaffnet/hesaffnet.py); the signature default 16 has no
        # checkpoint and no kernels here: refuse it where the user can see it, not at the first forward
        if PS != 32:
            raise L.AffnetB200Error("OriNetFast: the CUDA kernels are built for PS=32 (the shipped OriNet.pth); construct OriNetFast(PS=32)")
        k = int(PS / 4)
        self.features = make_features(AFF_CFG, [nn.Dropout(0.25), nn.Conv2d(64, 2, kernel_size=k, stride=1, padding=1, bias=True),
                                                nn.Tanh(), nn.AdaptiveAvgPool2d(1)])
        self.PS = PS
        self.halfPS = int(PS / 4)

    def forward(self, input, return_rot_matrix=True):
        x = self._check_input(input)
        n = x.size(0)
        R = torch.empty(n, 2, 2, dtype=torch.float32, device=x.device) if return_rot_matrix else None
        ang = None if return_rot_matrix else torch.empty(n, dtype=torch.float32, device=x.device)
        if n == 0:
            return R if return_rot_matrix else ang
        ws, nbytes = self._workspace(n, x.device)
        L.check(L.lib().ag_orinet_forward(self.handle(), L.ptr(x), n, None, 0, L.ptr(R), L.ptr(ang), L.ptr(ws), nbytes, L.stream_ptr()))
        return R if return_rot_matrix else ang

    def forward_raw(self, input):
        """The TorchScript export's contract (convertJIT/OriNetJIT.pt): the mean of tanh(head) over the 3x3 map -> [n,2]."""
        x = self._check_input(input)
        n = x.size(0)
        out = torch.empty(n, 2, dtype=torch.float32, device=x.device)
        if n:
            ws, nbytes = self._workspace(n, x.device)
            L.check(L.lib().ag_orinet_forward_raw(self.handle(), L.ptr(x), n, L.ptr(out), L.ptr(ws), nbytes, L.stream_ptr()))
        return out
