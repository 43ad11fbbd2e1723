"""GPU tests (-m gpu): the kernel paths that run when a default cannot must give the SAME BITS as the defaults.

- A driver without the tensor-map encoder (AG_BLUR_NO_TMA): the blur takes row-wise bulk copies.  The switch is read once per
  process, so the variant runs in a subprocess on the same seeded inputs and its pyramid / keypoints are compared with this process's.
- A pyramid whose levels lie 2^31 floats or more apart: the detector addresses them with 64-bit element offsets.  The pyramid is
  copied into one large buffer with octave 0's last level moved to float offset 2^31, where 32-bit offsets would overflow."""
import os
import subprocess
import sys

import pytest
import torch

import detect_cases as DC
import test_gpu_detect_nonfinite as NF
from helpers import Detector, adversarial_pyramid, flat_pyramid, gpu_pyramids, mixed_batch

pytestmark = pytest.mark.gpu

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
FAR = 1 << 31                  # float offset of octave 0's level 4 in the wide layout
WIDE = FAR + (1 << 26)         # floats of the wide buffer: room for that level of every case below


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


_SCRIPT = r"""
import ctypes as C, sys, torch
sys.path.insert(0, sys.argv[2]); sys.path.insert(0, sys.argv[2] + "/tests")
import affnet_b200._lib as L
from affnet_b200.HandCraftedModules import ScalePyramid
g = torch.Generator().manual_seed(11)
x = torch.rand(2, 1, 480, 640, generator=g) * 255
k = torch.ones(1, 1, 5, 5) / 25
x = torch.nn.functional.conv2d(x, k, padding=2).cuda().contiguous()      # smooth enough to have stable extrema
sp = ScalePyramid(3, 1.6, 5)
plan, buf = sp.build(x)
lib = L.lib()
cap = 65536
ws_buf = torch.empty(lib.ag_detect_ws_bytes(C.byref(plan), cap), dtype=torch.uint8, device="cuda")
ws = L.DetectWs()
L.check(lib.ag_detect_ws_carve(C.byref(plan), cap, L.ptr(ws_buf), C.byref(ws)))
L.check(lib.ag_detect(C.byref(plan), L.ptr(buf), 0.0, 5, C.byref(ws), L.stream_ptr()))
nf = 1500
resp = torch.zeros(2, nf, device="cuda"); lafs = torch.zeros(2, nf, 2, 3, device="cuda")
oc = torch.zeros(2, nf, dtype=torch.int32, device="cuda"); lv = torch.zeros(2, nf, dtype=torch.int32, device="cuda")
cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
L.check(lib.ag_select_keypoints(C.byref(plan), C.byref(ws), nf, 5.192, nf, L.ptr(resp), L.ptr(lafs), L.ptr(oc), L.ptr(lv), L.ptr(cnt), L.stream_ptr()))
torch.cuda.synchronize()
c = cnt.cpu()
for b in range(2):
    resp[b, int(c[b]):] = 0; lafs[b, int(c[b]):] = 0; oc[b, int(c[b]):] = 0; lv[b, int(c[b]):] = 0
torch.save({"pyr": buf.cpu(), "resp": resp.cpu(), "lafs": lafs.cpu(), "oc": oc.cpu(), "lv": lv.cpu(), "cnt": c}, sys.argv[1])
"""


def _run(tmp_path, name, env_extra):
    out = str(tmp_path / (name + ".pt"))
    env = dict(os.environ)
    env.pop("AG_BLUR_NO_TMA", None)
    env.update(env_extra)
    r = subprocess.run([sys.executable, "-c", _SCRIPT, out, ROOT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return torch.load(out)


def test_fallback_kernels_give_the_same_bits(tmp_path):
    base = _run(tmp_path, "default", {})
    assert int(base["cnt"].min()) > 200, base["cnt"]          # the input does produce keypoints
    other = _run(tmp_path, "blur_rowwise_bulk", {"AG_BLUR_NO_TMA": "1"})
    for key in base:
        assert torch.equal(base[key], other[key]), key


# ---- pyramids beyond 2^31 floats ----------------------------------------------------------------------------------------------------
def fits32(plan):
    """ag_detect's rule for 32-bit element offsets from each octave's first level."""
    for o in range(plan.n_octaves):
        offs = [plan.level_offset[o][d] - plan.level_offset[o][0] for d in range(5)]
        if min(offs) < -(1 << 30) or max(offs) + plan.B * plan.h[o] * plan.w[o] >= (1 << 31) - 64:
            return False
    return True


def wide_layout(L, plan, compact, buf):
    """Copy the pyramid `compact` (laid out by `plan`) into `buf`: every level at its own offset except octave 0's level 4, which goes
    to FAR; its usual place holds NaN.  -> the plan of the copy."""
    wide = L.PyramidPlan.from_buffer_copy(plan)
    n, src = plan.B * plan.h[0] * plan.w[0], plan.level_offset[0][4]
    buf[:plan.total_floats].copy_(compact[:plan.total_floats])
    buf[FAR:FAR + n].copy_(compact[src:src + n])
    buf[src:src + n].fill_(float("nan"))
    wide.level_offset[0][4] = FAR
    wide.total_floats = FAR + n
    return wide


def wide_cases(L):
    """(name, plan, compact pyramid buffer, NMS border, selections): the level-drop and odd-shape batches at nf 1, 40 and 0, the seam
    pyramid at border 0 and the k = 66 low-contrast pyramid at a_scale 5.192, and the non-finite batches (NaN / inf in the image or in
    single levels) at borders 5 and 0.  A selection is (kind, nf, out_cap, a_scale); kind "all" is ag_select_all_keypoints."""
    plan, buf, _ = gpu_pyramids(L, mixed_batch(97, 131, 5), 3)
    plan8 = L.make_plan(8, 40, 40, 3, 1.6, 5)
    planS = L.make_plan(1, *DC.SEAM_SHAPE, 3, 1.6, 5)
    planL = L.make_plan(1, 160, 200, 3, 1.6, 5)
    planN, bufN, pyrsN = gpu_pyramids(L, NF.seam_batch(), 3)
    top = [("top", 1, 1, 1.0), ("top", 40, 40, 1.0), ("top", 0, 4096, 1.0)]
    exact = [("top", 2000, None, 5.192)]
    nonfinite = [("top", 1, 1, 1.0), ("top", 40, 40, 1.0), ("all", 0, 4096, 1.0)]
    cases = [("odd", plan, buf, 5.192, top + exact),
             ("adv", plan8, flat_pyramid(plan8, [adversarial_pyramid(s) for s in range(8)]), 5.192, top + exact),
             ("seam", planS, flat_pyramid(planS, [DC.seam_case()[2]]), 0.0, exact),
             ("low66", planL, flat_pyramid(planL, [DC.scaled(DC.low_contrast_case()[2], 66)]), 5.192, exact)]
    for name, b in (("image", bufN), ("levels", flat_pyramid(planN, NF.level_pokes(pyrsN, 5)))):
        cases += [("%s border %d" % (name, mr), planN, b, float(mr), nonfinite) for mr in (5, 0)]
    return cases


def selections(det, sels):
    return [det.checked_select(nf, cap, a) if kind == "top" else det.select_all(cap, a) for kind, nf, cap, a in sels]


def same_bits(x, y):
    return torch.equal(x.view(torch.int32), y.view(torch.int32)) if x.is_floating_point() else torch.equal(x, y)


@pytest.fixture(scope="module")
def wide_buf():
    need, free = WIDE * 4, torch.cuda.mem_get_info()[0]
    if free < need + (1 << 29):
        pytest.skip("the wide pyramid layout needs %.2f GiB of free device memory, %.2f GiB are free" % (need / 2 ** 30, free / 2 ** 30))
    buf = torch.empty(WIDE, dtype=torch.float32, device="cuda")
    yield buf
    del buf
    torch.cuda.empty_cache()


def test_pyramid_beyond_2_31_floats_gives_the_same_bits(L, wide_buf):
    rows = 0
    for name, plan, compact, mr, sels in wide_cases(L):
        cap = 3 * sum(plan.h[o] * plan.w[o] for o in range(plan.n_octaves))
        wide = wide_layout(L, plan, compact, wide_buf)
        assert fits32(plan) and not fits32(wide), name
        want = selections(Detector(L, plan, compact, mr=mr, cap=cap), sels)
        dets = []
        names = [n for n, _ in L.profile(lambda: dets.append(Detector(L, wide, wide_buf, mr=mr, cap=cap)))]
        assert names.count("detect_rows_kernel") == 1, (name, names)
        got = selections(dets[0], sels)
        for sel, x, y in zip(sels, want, got):
            for i, (a, b) in enumerate(zip(x, y)):
                assert same_bits(a, b), (name, sel, i)
        assert max(int(x[4].max()) for x in want) > 0, name
        rows += sum(int(x[4].clamp(min=0).sum()) for x in want)
    print("\ndetector with levels 2^31 floats apart: %d keypoint rows bit-identical to the compact layout" % rows)
