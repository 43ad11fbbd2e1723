"""CPU tests of the SIFT descriptor (SIFTNet, pytorch_sift.py): the oracle against the reference's golden descriptors, ag_sift_windows
against the reference's windows, the SIFTNet wrapper's refusals, ag_pipeline_create_desc's refusals and workspace, and the oracle's
graf 1 <-> 6 application counts with SIFT as the descriptor.  No device code runs."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

import affnet_oracle as O
import oracle_sift as OS
from helpers import gold, gray_from_rgb, load_weights

W = load_weights()
SIFT_PS = (16, 32, 41, 65)
SETS = ("random", "graf", "constructed")


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        lib.build()
    lib.lib()
    return lib


@pytest.mark.parametrize("PS", SIFT_PS)
def test_oracle_matches_the_reference_descriptors(PS):
    """Measured: max |oracle - reference| = 0 on every set at every PS (same fp32 operations on the same CPU)."""
    z = gold("sift.npz")
    for name in SETS:
        d = OS.sift_describe(OS.golden_patches(z, name, PS))
        err = (d - torch.from_numpy(z["%s_desc_%d" % (name, PS)])).abs().max().item()
        print("PS %d %s: max |d| = %.3g" % (PS, name, err))
        assert d.shape[1] == 128 and err <= 1e-6, (name, err)


def test_constructed_patches_exercise_their_edges():
    """The constructed set is what it claims: flat patches (magnitude sqrt(1e-10), angle atan2(0, 1e-8) = 0) and the rising horizontal
    ramp put everything in angle bin 0, the falling one (on the +-pi cut: o = 12) in bin 4, and on the ramp with noise the clip binds on
    most cells (the clipped entries share the row's maximum)."""
    z = gold("sift.npz")
    d = torch.from_numpy(z["constructed_desc_32"]).view(-1, 8, 16)
    for r, b in ((0, 0), (1, 0), (2, 0), (3, 4), (8, 0)):
        energy = (d[r] ** 2).sum(dim=1)
        assert energy.argmax().item() == b and energy[b] > 0.9 * energy.sum(), r
    assert (d[8] == d[8].max()).sum() >= 10


@pytest.mark.parametrize("PS", SIFT_PS)
def test_sift_windows_are_the_reference_windows(L, PS):
    z = gold("sift.npz")
    gk, pk = np.zeros(PS * PS, np.float32), np.zeros(25 * 25, np.float32)
    k, s = C.c_int(), C.c_int()
    assert L.lib().ag_sift_windows(PS, gk.ctypes.data_as(C.c_void_p), pk.ctypes.data_as(C.c_void_p), C.byref(k), C.byref(s)) == 0
    assert (k.value, s.value) == (int(z["k_%d" % PS]), int(z["stride_%d" % PS]))
    kk = k.value
    assert np.array_equal(gk.reshape(PS, PS), z["gk_%d" % PS]) and np.array_equal(pk[:kk * kk].reshape(kk, kk), z["pk_%d" % PS])
    ogk, opk = OS.sift_windows(PS)
    assert np.array_equal(ogk.numpy(), z["gk_%d" % PS]) and np.array_equal(opk.numpy(), z["pk_%d" % PS])


def test_sift_windows_refuse_unsupported_patch_sizes(L):
    supported = []
    for PS in range(1, 80):
        k, s = OS.sift_geometry(PS)
        grid4 = 16 <= PS <= 65 and (PS - k) // s + 1 == 4
        rc = L.lib().ag_sift_windows(PS, None, None, None, None)
        assert (rc == 0) == grid4, PS
        if rc:
            assert L.lib().ag_last_error().decode().startswith("ag_sift_windows: unsupported patch size")
        else:
            supported.append(PS)
    assert [p for p in range(16, 66) if p not in supported] == [17, 18, 23, 28, 38, 48, 58]
    for PS in (15, 17, 28, 66):
        assert L.lib().ag_sift_windows(PS, None, None, None, None) == -1


def test_siftnet_wrapper(L):
    from affnet_b200.pytorch_sift import SIFTNet
    s = SIFTNet()
    assert s.PS == 65 and (s.bin_weight_kernel_size, s.bin_weight_stride) == (25, 13) and s.gk.shape == (65, 65)
    assert abs(s.gk[32, 32].item() - math.exp(-0.5 / (0.9 * 32.5 ** 2))) < 1e-7     # the centre of an odd window is 32.5
    for kw in (dict(num_ang_bins=16), dict(num_spatial_bins=3)):
        with pytest.raises(L.AffnetB200Error, match="num_ang_bins=8 and num_spatial_bins=4"):
            SIFTNet(32, **kw)
    with pytest.raises(L.AffnetB200Error, match="unsupported patch size"):
        SIFTNet(28)
    with pytest.raises(L.AffnetB200Error, match="CUDA tensor"):
        SIFTNet(32)(torch.zeros(2, 1, 32, 32))


# ---- ag_pipeline_create_desc ---------------------------------------------------------------------------------------------------------
class FakeNets:
    """Non-NULL net handles: create_desc stores the borrowed pointers and never dereferences them at create time."""

    def __init__(self):
        self._buf = (C.c_char * 64)()
        self.h = C.c_void_p(C.addressof(self._buf))


def cfg_of(L, K=300, do_ori=1, B=2, H=240, Wd=320):
    return L.PipelineConfig(B, H, Wd, K, 3, 5, 1.6, 5.192, do_ori, 0)


def create(L, cfg, est, desc, aff, ori, hard):
    h = C.c_void_p()
    if desc is None:
        rc = L.lib().ag_pipeline_create_ex(C.byref(cfg), C.byref(est), aff, ori, hard, C.byref(h))
    else:
        rc = L.lib().ag_pipeline_create_desc(C.byref(cfg), C.byref(est), C.byref(desc), aff, ori, hard, C.byref(h))
    nbytes = L.lib().ag_pipeline_workspace_bytes(h) if rc == 0 else 0
    if rc == 0:
        L.lib().ag_pipeline_destroy(h)
    return rc, L.lib().ag_last_error().decode() if rc else "", nbytes


def test_create_desc_refusals_and_error_texts(L):
    f = FakeNets().h
    E, D = L.PipelineEstimators, L.PipelineDescriptor
    est = E(L.SHAPE_AFFNET, 1, 0, L.ORI_HISTOGRAM, 19)
    cases = [
        (D(2, 32, 0.2), f, "unknown descriptor kind"),
        (D(-1, 32, 0.2), f, "unknown descriptor kind"),
        (D(L.DESC_HARDNET, 65, 0.2), f, "AG_DESC_HARDNET needs ps = 32"),
        (D(L.DESC_HARDNET, 32, 0.2), None, "AG_DESC_HARDNET needs a HardNet"),
        (D(L.DESC_SIFT, 28, 0.2), None, "AG_DESC_SIFT: unsupported ps"),
        (D(L.DESC_SIFT, 66, 0.2), None, "AG_DESC_SIFT: unsupported ps"),
        (D(L.DESC_SIFT, 32, 0.0), None, "AG_DESC_SIFT: clipval must be finite and positive"),
        (D(L.DESC_SIFT, 32, -0.2), None, "AG_DESC_SIFT: clipval must be finite and positive"),
        (D(L.DESC_SIFT, 32, float("nan")), None, "AG_DESC_SIFT: clipval must be finite and positive"),
        (D(L.DESC_SIFT, 32, float("inf")), None, "AG_DESC_SIFT: clipval must be finite and positive"),
    ]
    for desc, hard, text in cases:
        rc, msg, _ = create(L, cfg_of(L), est, desc, f, None, hard)
        assert rc == -1 and text in msg and msg.startswith("ag_pipeline_create_desc: "), (rc, msg, text)
    # the estimator rules are unchanged and name create_desc
    rc, msg, _ = create(L, cfg_of(L), E(L.SHAPE_AFFNET, 1, 0, L.ORI_ORINET, 0), D(L.DESC_SIFT, 32, 0.2), f, None, None)
    assert rc == -1 and msg == "ag_pipeline_create_desc: AG_ORI_ORINET needs an OriNet"
    # SIFT needs no HardNet; every supported SIFT patch size is accepted
    for ps in (16, 32, 41, 65):
        assert create(L, cfg_of(L), est, D(L.DESC_SIFT, ps, 0.2), f, None, None)[0] == 0, L.lib().ag_last_error()


def test_create_desc_workspace(L):
    f = FakeNets().h
    E, D = L.PipelineEstimators, L.PipelineDescriptor
    lib = L.lib()
    B, K = 2, 300
    M = int(1.5 * K)
    al = lambda n: (n + 255) // 256 * 256  # noqa: E731
    hb = lib.ag_net_workspace_bytes(L.NET_HARDNET, B * K)
    ab = lib.ag_net_workspace_bytes(L.NET_AFFNET, B * M)
    ob = lib.ag_net_workspace_bytes(L.NET_ORINET, B * K)
    modes = [
        (cfg_of(L, K=K, B=B), E(L.SHAPE_AFFNET, 1, 0, L.ORI_ORINET, 0), max(ab, ob)),
        (cfg_of(L, K=K, B=B), E(L.SHAPE_AFFNET, 1, 0, L.ORI_HISTOGRAM, 19), ab),
        (cfg_of(L, K=K, B=B), E(L.SHAPE_NONE, 0, 0, L.ORI_ORINET, 0), ob),
        (cfg_of(L, K=K, B=B), E(L.SHAPE_BAUMBERG, 16, 19, L.ORI_HISTOGRAM, 19), 0),
        (cfg_of(L, K=K, B=B), E(L.SHAPE_NONE, 0, 0, L.ORI_HISTOGRAM, 19), 0),
        (cfg_of(L, K=K, B=B, do_ori=0), E(L.SHAPE_NONE, 0, 0, L.ORI_NONE, 0), 0),
    ]
    for cfg, est, nets in modes:
        rc, _, ex = create(L, cfg, est, None, f, f, f)
        rc2, _, hard = create(L, cfg, est, D(L.DESC_HARDNET, 32, 0.2), f, f, f)
        assert rc == rc2 == 0 and ex == hard          # create_ex is create_desc with {HARDNET, 32}
        for ps in (32, 65):
            rc3, msg, sift = create(L, cfg, est, D(L.DESC_SIFT, ps, 0.2), f, f, None)
            assert rc3 == 0, msg
            # the net share shrinks from max(nets, HardNet) to the shape / orientation nets alone (none at all for the hand-crafted modes)
            assert sift == hard - al(max(nets, hb)) + al(nets), (est.shape, est.ori, ps)
            assert sift < hard or nets >= hb   # AffNet's share (1.5 K rows) already covers HardNet's: no saving there
            if nets == 0:
                assert sift == hard - al(hb)


def test_oracle_graf_1_to_6_application_counts_with_sift():
    """The reference's application check with SIFTNet(32) in place of HardNet (golden: the unmodified reference) from the oracle
    restatement, within 2 (the slack the HardNet version allows with the gradient-histogram orientation).  Measured: 300 tentatives
    against the reference's 302 without orientation, because SIFT's ratio test has near-ties that HardNet's has not: seven rows of that
    pair lie within 1e-3 of the 0.8 threshold, so the oracle's pyramid and sampler rounding moves two of them across it."""
    z, f, s = gold("graf_match.npz"), gold("graf_full.npz"), gold("sift.npz")
    x1, x6 = gray_from_rgb(f["rgb"]), gray_from_rgb(z["rgb6"])
    for mode in ("hcori", "noori"):
        out = []
        for x in (x1, x6):
            dL, _, st = O.detect(x, W["affnet"], None, num_features=int(s["K"]), do_ori=mode != "noori")
            d, _, _ = OS.describe_sift(dL, st, 32)
            out.append((dL, d))
        tent, true = O.match_and_verify(out[0][0], out[0][1], out[1][0], out[1][1], torch.from_numpy(z["H1to6"]), float(s["snn"]),
                                        float(s["px"]))
        print(mode, tent, true, "golden", int(s[mode + "_tent"]), int(s[mode + "_true"]))
        slack = 2
        assert abs(tent - int(s[mode + "_tent"])) <= slack and abs(true - int(s[mode + "_true"])) <= slack, (mode, tent, true)
