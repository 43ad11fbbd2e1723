"""CPU tests (-m "not gpu"): the C-ABI library loads, exports every symbol include/affnet_b200.h declares, and its
host-side logic (pyramid plan, argument validation, error reporting) agrees with the oracle.  No compute calls."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import affnet_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        lib.build()
    lib.lib()
    return lib


def test_every_header_symbol_is_exported_and_bound(L):
    hdr = open(os.path.join(ROOT, "include", "affnet_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = set(re.findall(r"\b(ag_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) >= 30
    raw = C.CDLL(L.LIB_PATH)
    for n in sorted(names):
        assert hasattr(raw, n), "header declares %s but the .so does not export it" % n
        assert n in L.PROTOTYPES, "%s has no ctypes prototype" % n
    assert set(L.PROTOTYPES) == names
    assert L.lib().ag_abi_version() == 1


@pytest.mark.parametrize("H,W,border", [(640, 800, 5), (768, 1024, 5), (1080, 1920, 5), (2160, 3840, 33), (256, 320, 5), (65, 77, 16), (30, 30, 5)])
def test_pyramid_plan_matches_oracle(L, H, W, border):
    sizes, bs, sig, pix = O.pyramid_plan(H, W, 3, 1.6, border)
    p = L.make_plan(2, H, W, 3, 1.6, border)
    assert p.n_octaves == len(sizes) and p.n_levels == 5
    off = 0
    for o in range(p.n_octaves):
        assert (p.h[o], p.w[o]) == sizes[o] and p.pix_dist[o] == pix[o][0]
        for l in range(5):
            assert p.sigma[o][l] == sig[o][l]                    # bit-identical python-float arithmetic
            assert p.blur_sigma[o][l] == (bs[o][l] or 0.0)
            assert p.level_offset[o][l] == off
            off += 2 * sizes[o][0] * sizes[o][1]
    assert p.total_floats == off
    if (H, W, border) == (2160, 3840, 33):
        assert p.n_octaves == 5                                   # BASELINE config 5: the "5-octave" pyramid


def test_argument_validation_and_error_text(L):
    lib = L.lib()
    p = L.PyramidPlan()
    assert lib.ag_pyramid_plan(1, 0, 10, 3, 1.6, 5, C.byref(p)) == -1
    assert b"bad image size" in lib.ag_last_error()
    assert lib.ag_pyramid_plan(1, 64, 64, 9, 1.6, 5, C.byref(p)) == -1
    assert lib.ag_net_blob_floats(7) == 0
    with pytest.raises(L.AffnetB200Error):
        L.check(lib.ag_gaussian_blur(None, None, 1, 8, 8, 1.0, None))
    blob = np.zeros(10, np.float32)
    h = C.c_void_p()
    assert lib.ag_net_create(0, blob.ctypes.data_as(C.c_void_p), 10, C.byref(h)) == -1
    assert b"blob has 10 floats" in lib.ag_last_error()


def test_debug_probe_refusals(L):
    """The developer diagnostics refuse NULL arguments before any CUDA call, naming themselves; an empty probe is a no-op."""
    lib = L.lib()
    buf = np.zeros(4, np.float32)
    p = buf.ctypes.data_as(C.c_void_p)
    assert "ag_debug_tanhf" in L.PROTOTYPES
    for x, y in ((None, p), (p, None), (None, None)):
        assert lib.ag_debug_tanhf(x, 4, y, None) == -1
        assert lib.ag_last_error() == b"ag_debug_tanhf: NULL argument"
    assert lib.ag_debug_tanhf(None, 0, None, None) == -1              # NULL is refused before the size is looked at
    assert lib.ag_debug_tanhf(p, 0, p, None) == 0 and lib.ag_debug_tanhf(p, -3, p, None) == 0
    assert lib.ag_debug_tcx_layer(None, p, 1, 1, p, p, 1 << 20, None) == -1
    assert lib.ag_last_error() == b"ag_debug_tcx_layer: NULL argument"
    assert lib.ag_debug_libm(p, p, 4, p, None, p, None) == -1
    assert lib.ag_last_error() == b"ag_debug_libm: NULL argument"


def test_blob_sizes_match_checkpoints(L):
    from helpers import load_weights
    W = load_weights()
    for kind, name in ((0, "affnet"), (1, "orinet"), (2, "hardnet")):
        assert L.lib().ag_net_blob_floats(kind) == sum(v.numel() for v in W[name].values())


def test_no_cpu_fallback(L):
    """The product refuses CPU tensors instead of silently computing elsewhere."""
    from affnet_b200.architectures import AffNetFast
    from affnet_b200.LAF import extract_patches
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    with pytest.raises(L.AffnetB200Error):
        AffNetFast(PS=32).eval()(torch.zeros(2, 1, 32, 32))
    with pytest.raises(L.AffnetB200Error):
        extract_patches(torch.zeros(1, 1, 8, 8), torch.zeros(1, 2, 3))
    with pytest.raises(L.AffnetB200Error):
        ScaleSpaceAffinePatchExtractor(num_features=10)(torch.zeros(1, 1, 64, 64))


def test_product_does_not_import_oracle():
    import glob
    for f in glob.glob(os.path.join(ROOT, "affnet_b200", "**", "*.py"), recursive=True) + glob.glob(os.path.join(ROOT, "affnet_b200", "csrc", "*")):
        if os.path.isfile(f) and not f.endswith((".o", ".log", ".so")):
            src = open(f, errors="ignore").read()
            assert "affnet_oracle" not in src and "ref_harness" not in src, f


def test_modules_keep_reference_interface(L):
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    from helpers import load_weights
    W = load_weights()
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])   # checkpoint key names
    assert a.PS == 32 and o.PS == 32
    d = ScaleSpaceAffinePatchExtractor(mrSize=5.192, num_features=2000, border=5, num_Baum_iters=1, AffNet=a)
    assert d.num == 2000 and d.th == 0
    d = ScaleSpaceAffinePatchExtractor(th=-1, num_features=2000)
    assert d.num == -1 and d.th == -1                               # SparseImgRepresenter.py:33-37
    for m in ("forward", "multiScaleDetector", "getAffineShape", "getOrientation", "extract_patches_from_pyr"):
        assert callable(getattr(d, m))


def test_host_lafs2ell_matches_reference_golden():
    """a17: the host-side output format LAFs2ell (LAF.py:225-240, float64 numpy SVD) against rows produced by the unmodified
    reference (tests/golden/make_golden.py::make_ell), plus the text file layout of hesaffnet.py:56-60."""
    import numpy as np
    from helpers import gold
    from affnet_b200.LAF import LAFs2ell
    z = gold("ell.npz")
    lafs = z["lafs"][z["host_rows"]]
    e = LAFs2ell(lafs)
    g = z["ell_host"]
    assert e.shape == g.shape == (len(lafs), 5) and e.dtype == np.float64
    assert np.array_equal(e[:, :2], g[:, :2])
    assert np.allclose(e[:, 2:], g[:, 2:], rtol=1e-6, atol=0)       # same float32 SVD as the reference (LAPACK build may differ in the last bit)
    assert LAFs2ell(np.zeros((0, 2, 3))).shape == (0, 5)


def test_helpers_synthetic_image_is_the_oracles():
    """bench.py's product arm takes its inputs from tests/helpers.py so that it imports nothing from oracle/: same bits as the oracle's generator."""
    import torch
    import affnet_oracle as O
    from helpers import synthetic_image
    assert torch.equal(synthetic_image(96, 131, 7), O.synthetic_image(96, 131, 7))


def test_orinet_signature_default_is_refused_at_construction():
    """OriNetFast(PS=16) is the reference's signature default (architectures.py:33-35) but has neither checkpoint nor kernels: the
    constructor refuses it (every caller of the reference passes PS=32), instead of failing at the first forward."""
    import pytest as _pt
    from affnet_b200 import _lib as L
    from affnet_b200.architectures import OriNetFast
    with _pt.raises(L.AffnetB200Error):
        OriNetFast()
    assert OriNetFast(PS=32).PS == 32
