"""CPU tests (-m "not gpu") of the batched SNN matcher: the host-side refusals of ag_match_pairs (checked before any CUDA call) and their
texts, its workspace size, the refusals of Losses.match_snn_pairs, and the expected-value rule of the GPU tests (snn_rule.snn_expected)
pinned to the oracle's match_snn."""
import ctypes as C
import os

import pytest
import torch

import affnet_oracle as O
from snn_rule import snn_expected


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        lib.build()
    lib.lib()
    return lib


def _ws(S1, cap1, S2, cap2, P):
    up = lambda x: (x + 255) // 256 * 256  # noqa: E731
    return up(S1 * cap1 * 4) + up(S2 * cap2 * 4) + up(P * cap2)


def test_workspace_bytes(L):
    lib = L.lib()
    for args in ((1, 1, 1, 1, 1), (16, 2000, 16, 2000, 240), (64, 4000, 64, 4000, 63), (1, 16384, 1, 12000, 1), (3, 700, 5, 333, 1000)):
        assert lib.ag_match_pairs_workspace_bytes(*args) == _ws(*args), args
    assert lib.ag_match_pairs_workspace_bytes(1, 16384, 1, 12000, 1) < 200 * 1024   # no n1 x n2 matrix (that would be 750 MiB)
    for bad in ((0, 1, 1, 1, 1), (1, 0, 1, 1, 1), (1, 1, 0, 1, 1), (1, 1, 1, 0, 1), (1, 1, 1, 1, 0)):
        assert lib.ag_match_pairs_workspace_bytes(*bad) == 0
    # the single-pair matcher is the batched one with S = P = 1
    assert lib.ag_match_snn_workspace_bytes(700, 733) == _ws(1, 700, 1, 733, 1)


def test_refusals_and_texts(L):
    """Every refusal returns before any CUDA call (the pointers below are never dereferenced) and names ag_match_pairs."""
    lib = L.lib()
    f = C.c_void_p(256)   # a non-NULL stand-in for device memory

    def call(d1=f, S1=2, cap1=10, d2=f, S2=2, cap2=10, dim=128, pairs=None, P=2, ws=f, nb=1 << 20, outs=(f, f, f, f)):
        return lib.ag_match_pairs(d1, None, S1, cap1, d2, None, S2, cap2, dim, pairs, P, 0.8, ws, nb, *outs, None, None, None)

    def refused(rc, code, text):
        assert rc == code
        msg = lib.ag_last_error().decode()
        assert msg.startswith("ag_match_pairs") and text in msg, msg

    for kw in (dict(d1=None), dict(d2=None), dict(ws=None), dict(outs=(None, f, f, f)), dict(outs=(f, None, f, f)), dict(outs=(f, f, None, f)),
               dict(outs=(f, f, f, None))):
        refused(call(**kw), -1, "NULL")
    for kw in (dict(dim=0), dict(S1=0), dict(S2=0), dict(cap1=0), dict(cap2=-3), dict(P=0), dict(pairs=f, P=-1)):
        refused(call(**kw), -1, "must be >= 1")
    refused(call(S1=3, P=3), -1, "S1 == S2 == P")
    refused(call(P=3), -1, "S1 == S2 == P")
    refused(call(cap1=4194241), -1, "cap1 above 4194240")
    need = _ws(2, 10, 2, 10, 2)
    refused(call(nb=need - 1), -3, "workspace too small (%d bytes, needs %d)" % (need - 1, need))
    refused(call(pairs=f, S1=3, S2=5, P=7, nb=_ws(3, 10, 5, 10, 7) - 1), -3, "workspace too small")
    # ag_match_snn keeps its own refusals
    assert lib.ag_match_snn(f, 0, f, 3, 128, 0.8, f, 1 << 20, f, f, f, f, None) == -1 and b"ag_match_snn" in lib.ag_last_error()
    assert lib.ag_match_snn(f, 5, f, 3, 128, 0.8, f, 1, f, f, f, f, None) == -3
    assert lib.ag_last_error() == b"ag_match_snn: workspace too small"


def test_wrapper_refusals(L):
    from affnet_b200.Losses import match_snn_pairs
    d = torch.zeros(2, 5, 8)
    cases = [
        (dict(desc1=torch.zeros(5, 8)), "desc1 must be [S,cap,D]"),
        (dict(desc1=d, desc2=torch.zeros(5, 8)), "desc2 must be [S,cap,D]"),
        (dict(desc1=d, desc2=torch.zeros(2, 5, 7)), "different D"),
        (dict(desc1=d, count1=torch.zeros(3, dtype=torch.int32)), "count1 must be an integer tensor [2]"),
        (dict(desc1=d, count1=torch.zeros(2)), "count1 must be an integer tensor"),
        (dict(desc1=d, desc2=torch.zeros(3, 4, 8), count2=torch.zeros(2, dtype=torch.int32)), "count2 must be an integer tensor [3]"),
        (dict(desc1=d, desc2=torch.zeros(3, 4, 8)), "needs S1 == S2"),
        (dict(desc1=d, pairs=torch.zeros(4, 3, dtype=torch.int32)), "pairs must be an integer tensor [P,2]"),
        (dict(desc1=d, pairs=torch.zeros(4, dtype=torch.int32)), "pairs must be an integer tensor [P,2]"),
        (dict(desc1=d, pairs=torch.zeros(4, 2)), "pairs must be an integer tensor [P,2]"),
        (dict(desc1=d), "must be a CUDA tensor"),                                                   # CPU descriptors
        (dict(desc1=d, count1=torch.zeros(2, dtype=torch.int64)), "count1 must be a CUDA tensor"),  # CPU counts
        (dict(desc1=d, pairs=torch.zeros(4, 2, dtype=torch.int64)), "pairs must be a CUDA tensor"),  # CPU pairs
    ]
    for kw, text in cases:
        with pytest.raises(L.AffnetB200Error, match=text.replace("[", r"\[").replace("]", r"\]")):
            match_snn_pairs(**kw)


def _snn_8f_fixture():
    """The descriptors of test_gpu_parity.py::test_snn_matcher_8f."""
    g = torch.Generator().manual_seed(21)
    d1 = torch.nn.functional.normalize(torch.randn(700, 128, generator=g), dim=1)
    d2 = torch.cat([torch.nn.functional.normalize(d1[:400] + 0.25 * torch.randn(400, 128, generator=g), dim=1),
                    torch.nn.functional.normalize(torch.randn(333, 128, generator=g), dim=1)])
    return d1, d2


def test_expected_rule_is_the_oracles_match_snn():
    d1, d2 = _snn_8f_fixture()
    idx2, mn, sec, keep, tent = snn_expected(O.distance_matrix_vector(d1, d2), 0.8)
    o1, o2, omn, osec = O.match_snn(d1, d2, 0.8)
    _, oidx2 = torch.min(O.distance_matrix_vector(d1, d2), 1)
    assert torch.equal(idx2, oidx2) and torch.equal(mn, omn) and torch.equal(sec, osec)
    assert torch.equal(tent[:, 0], o1) and torch.equal(tent[:, 1], o2) and torch.equal(keep.nonzero().view(-1), o1)
    assert 0 < tent.size(0) < 700


def test_expected_rule_edges():
    """Lowest column among equal minima, NaN ignored (a NaN row gets (+inf, 0)), the 100000 mask and a single column."""
    nan, inf = float("nan"), float("inf")
    D = torch.tensor([[2.0, 1.0, 1.0, 3.0],
                      [nan, nan, nan, nan],
                      [nan, 5.0, 4.0, 4.0],
                      [1.5, 1.2, 9.0, 1.1]])
    idx2, mn, sec, keep, tent = snn_expected(D, 0.8)
    assert idx2.tolist() == [1, 0, 2, 3] and mn[0] == 1 and mn[1] == inf and mn[2] == 4 and mn[3] == 1.1
    # marked columns 0, 1, 2, 3: everything is 100000 except NaNs
    assert sec.tolist() == [100000.0] * 4
    D2 = torch.tensor([[1.0, 2.0, 3.0], [5.0, 0.5, 4.0]])
    idx2, mn, sec, keep, tent = snn_expected(D2, 0.8)
    assert idx2.tolist() == [0, 1] and sec.tolist() == [3.0, 4.0]      # row 0's second-nearest (column 1) is row 1's nearest: masked
    assert tent.tolist() == [[0, 0], [1, 1]]
    idx2, mn, sec, keep, tent = snn_expected(torch.tensor([[0.3], [0.2]]), 0.8)
    assert idx2.tolist() == [0, 0] and sec.tolist() == [100000.0, 100000.0] and keep.tolist() == [True, True]
