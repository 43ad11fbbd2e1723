"""CPU tests (-m "not gpu") of the top-K entry points at any count: ag_select_topk_keypoints, ag_affine_shape_filter_topk and
ag_pipeline_create_topk.  Their bindings, scratch sizes, refusals and error texts, and the pipeline's acceptance of K above the shared-memory
limit with the same workspace as ag_pipeline_create_desc below it.  Every call here returns before any CUDA call."""
import ctypes as C
import os

import pytest

NEW = ("ag_select_topk_workspace_bytes", "ag_select_topk_keypoints", "ag_affine_shape_filter_topk_workspace_bytes",
       "ag_affine_shape_filter_topk", "ag_pipeline_create_topk")
FAKE = C.c_void_p(256)   # a non-NULL device pointer that no call below dereferences


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        lib.build()
    lib.lib()
    return lib


def test_new_symbols_are_exported_and_bound(L):
    raw = C.CDLL(L.LIB_PATH)
    for n in NEW:
        assert hasattr(raw, n) and n in L.PROTOTYPES, n
        assert getattr(L.lib(), n).argtypes == L.PROTOTYPES[n][1]


def test_workspace_zero_below_the_limit_and_growing_above(L):
    lib = L.lib()
    for B in (1, 2, 5):
        plan = L.make_plan(B, 1080, 1920)
        cap = 1080 * 1920 // 8
        assert lib.ag_select_topk_workspace_bytes(C.byref(plan), cap, 1) == 0
        assert lib.ag_select_topk_workspace_bytes(C.byref(plan), cap, 16384) == 0
        assert lib.ag_affine_shape_filter_topk_workspace_bytes(B, 1) == 0
        assert lib.ag_affine_shape_filter_topk_workspace_bytes(B, 16384) == 0
        prev_s = prev_f = 0
        for n in (16385, 20000, 40000, 100000, 1 << 22):
            s = lib.ag_select_topk_workspace_bytes(C.byref(plan), cap, n)
            f = lib.ag_affine_shape_filter_topk_workspace_bytes(B, n)
            assert s >= prev_s and f >= prev_f and s >= B * n * 24 and f >= B * n * 29, (B, n, s, f)
            assert s % 256 == 0 and f % 256 == 0
            prev_s, prev_f = s, f
    plan = L.make_plan(1, 64, 64)
    assert lib.ag_select_topk_workspace_bytes(None, 100, 20000) == 0
    assert lib.ag_select_topk_workspace_bytes(C.byref(plan), 0, 20000) == 0
    assert lib.ag_affine_shape_filter_topk_workspace_bytes(0, 20000) == 0


def detect_ws(L, plan, cand_cap):
    ws = L.DetectWs()
    ws.B, ws.cand_cap, ws.n_level_slots = plan.B, cand_cap, plan.n_octaves * (plan.n_levels - 2)
    return ws


def select(L, plan, ws, nf, out_cap, scratch, nbytes, outs=None):
    outs = outs or [FAKE] * 5
    rc = L.lib().ag_select_topk_keypoints(C.byref(plan), C.byref(ws), nf, 1.0, out_cap, scratch, nbytes, *outs, None)
    return rc, L.lib().ag_last_error().decode() if rc else ""


def test_select_refusals_and_texts(L):
    plan = L.make_plan(2, 1080, 1920)
    ws = detect_ws(L, plan, 200000)
    need = L.lib().ag_select_topk_workspace_bytes(C.byref(plan), 200000, 20000)
    assert need > 0
    cases = [
        (20000, 20000, FAKE, need, [None, FAKE, FAKE, FAKE, FAKE], -1, "ag_select_topk_keypoints: NULL argument"),
        (20000, 20000, FAKE, need, [FAKE, FAKE, FAKE, FAKE, None], -1, "ag_select_topk_keypoints: NULL argument"),
        (20000, 20000, None, need, None, -1, "ag_select_topk_keypoints: NULL argument"),
        (20000, 0, FAKE, need, None, -1, "ag_select_topk_keypoints: out_cap must be positive"),
        (20000, 20000, FAKE, need - 1, None, -3, "ag_select_topk_keypoints: scratch of %d bytes needed, %d given" % (need, need - 1)),
        (20000, 20000, None, 0, None, -3, "ag_select_topk_keypoints: scratch of %d bytes needed, 0 given" % need),
        (0, 20000, FAKE, 0, None, -3, "scratch of %d bytes needed" % need),                 # num_features <= 0: out_cap decides
        (30000, 20000, FAKE, 0, None, -3, "scratch of %d bytes needed" % need),             # min(num_features, out_cap) decides
    ]
    for nf, out_cap, scratch, nbytes, outs, rc_want, text in cases:
        rc, msg = select(L, plan, ws, nf, out_cap, scratch, nbytes, outs)
        assert rc == rc_want and text in msg and msg.startswith("ag_select_topk_keypoints: "), (nf, out_cap, rc, msg)
    bad = detect_ws(L, plan, 200000)
    bad.B = 3
    rc, msg = select(L, plan, bad, 20000, 20000, FAKE, need)
    assert rc == -1 and msg == "ag_select_topk_keypoints: workspace / plan mismatch"
    # the old entry point keeps its limit and its text
    rc = L.lib().ag_select_keypoints(C.byref(plan), C.byref(ws), 20000, 1.0, 20000, *[FAKE] * 5, None)
    assert rc == -3 and L.lib().ag_last_error().decode().startswith("ag_select_keypoints: selecting 20000 keypoints needs")


def test_filter_refusals_and_texts(L):
    lib = L.lib()
    cap = 40000
    need = lib.ag_affine_shape_filter_topk_workspace_bytes(2, cap)

    def call(B, cap, out_cap, scratch, nbytes, first=FAKE):
        rc = lib.ag_affine_shape_filter_topk(first, FAKE, FAKE, FAKE, FAKE, FAKE, B, cap, 20000, out_cap, scratch, nbytes, *[FAKE] * 5, None)
        return rc, lib.ag_last_error().decode() if rc else ""

    assert call(2, cap, cap, FAKE, need, first=None) == (-1, "ag_affine_shape_filter_topk: NULL argument")
    assert call(2, cap, cap, None, need) == (-1, "ag_affine_shape_filter_topk: NULL argument")
    assert call(0, cap, cap, FAKE, need) == (-1, "ag_affine_shape_filter_topk: bad sizes")
    assert call(2, 0, cap, FAKE, need) == (-1, "ag_affine_shape_filter_topk: bad sizes")
    assert call(2, cap, 0, FAKE, need) == (-1, "ag_affine_shape_filter_topk: bad sizes")
    assert call(2, cap, cap, FAKE, need - 1) == (-3, "ag_affine_shape_filter_topk: scratch of %d bytes needed, %d given" % (need, need - 1))
    assert call(2, cap, 10, None, 0) == (-3, "ag_affine_shape_filter_topk: scratch of %d bytes needed, 0 given" % need)
    rc = lib.ag_affine_shape_filter(*[FAKE] * 6, 2, cap, 20000, cap, *[FAKE] * 5, None)
    assert rc == -3 and lib.ag_last_error().decode().startswith("ag_affine_shape_filter: cap 40000 needs")


class FakeNets:
    """A non-NULL net handle: pipeline creation stores the borrowed pointers and never dereferences them."""

    def __init__(self):
        self._buf = (C.c_char * 64)()
        self.h = C.c_void_p(C.addressof(self._buf))


def create(L, fn, K, est, B=2, H=1080, Wd=1920, desc=None):
    f = FakeNets()
    cfg = L.PipelineConfig(B, H, Wd, K, 3, 5, 1.6, 5.192, 1 if est.ori else 0, 0)
    desc = desc or L.PipelineDescriptor(L.DESC_HARDNET, 32, 0.2)
    h = C.c_void_p()
    rc = getattr(L.lib(), fn)(C.byref(cfg), C.byref(est), C.byref(desc), f.h, f.h, f.h, C.byref(h))
    if rc:
        return rc, L.lib().ag_last_error().decode(), 0
    n = L.lib().ag_pipeline_workspace_bytes(h)
    L.lib().ag_pipeline_destroy(h)
    return rc, "", n


MODES = {
    "affnet1-orinet": lambda L: L.PipelineEstimators(L.SHAPE_AFFNET, 1, 0, L.ORI_ORINET, 0),
    "affnet3-none": lambda L: L.PipelineEstimators(L.SHAPE_AFFNET, 3, 0, L.ORI_NONE, 0),
    "baumberg16-histogram": lambda L: L.PipelineEstimators(L.SHAPE_BAUMBERG, 16, 19, L.ORI_HISTOGRAM, 19),
    "none-orinet": lambda L: L.PipelineEstimators(L.SHAPE_NONE, 0, 0, L.ORI_ORINET, 0),
}


def test_pipeline_create_topk_accepts_any_k(L):
    shape, plain = MODES["affnet1-orinet"](L), MODES["none-orinet"](L)
    assert create(L, "ag_pipeline_create_desc", 10924, shape)[0] == -3
    assert create(L, "ag_pipeline_create_desc", 16385, plain)[0] == -3
    for K, est in ((10924, shape), (16385, plain), (20000, shape), (40000, plain), (20000, MODES["baumberg16-histogram"](L))):
        rc, msg, n = create(L, "ag_pipeline_create_topk", K, est)
        assert rc == 0 and n > 0, (K, msg)
    # the other refusals keep the entry point's name
    rc, msg, _ = create(L, "ag_pipeline_create_topk", 0, plain)
    assert rc == -1 and msg == "ag_pipeline_create_topk: num_features must be positive"
    rc, msg, _ = create(L, "ag_pipeline_create_topk", 300, L.PipelineEstimators(L.SHAPE_BAUMBERG, 1, 2, L.ORI_ORINET, 0))
    assert rc == -1 and msg == "ag_pipeline_create_topk: shape_ps out of range (3..41)"


@pytest.mark.parametrize("mode", sorted(MODES))
def test_pipeline_create_topk_equals_desc_within_the_limit(L, mode):
    """Same workspace bytes as ag_pipeline_create_desc wherever that accepts K; one scratch region more above, sized for the larger step."""
    est = MODES[mode](L)
    shape = est.shape != L.SHAPE_NONE
    sift = L.PipelineDescriptor(L.DESC_SIFT, 32, 0.2)
    Ks = (1, 300, 2000, 10923) if shape else (1, 2000, 10923, 16384)
    for K in Ks:
        for desc in (None, sift):
            a, b = create(L, "ag_pipeline_create_desc", K, est, desc=desc), create(L, "ag_pipeline_create_topk", K, est, desc=desc)
            assert a[0] == 0 and b[0] == 0 and a[2] == b[2], (mode, K, a, b)
    plan = L.make_plan(2, 1080, 1920)
    al = lambda n: (n + 255) // 256 * 256  # noqa: E731
    K = 10924 if shape else 16385
    M = int(1.5 * K) if shape else K
    big = create(L, "ag_pipeline_create_topk", K, est)[2]
    sb = L.lib().ag_select_topk_workspace_bytes(C.byref(plan), 1080 * 1920 // 8, M)
    fb = L.lib().ag_affine_shape_filter_topk_workspace_bytes(2, M) if shape else 0
    assert sb > 0 and big >= al(max(sb, fb))
