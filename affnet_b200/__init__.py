"""affnet_b200: H100-native (sm_90a) HesAffNet + HardNet detect-and-describe hot path.

Drop-in mirror of the reference's Python entry points (ducha-aiki/affnet):
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.LAF import extract_patches, denormalizeLAFs, normalizeLAFs
All compute goes through the C ABI in include/affnet_b200.h (affnet_b200/lib/libaffnet_b200.so).
"""
from . import _lib  # noqa: F401

__all__ = ["_lib"]
