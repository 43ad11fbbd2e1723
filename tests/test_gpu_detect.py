"""GPU tests (-m gpu) of the detector stage alone: `ag_detect` (Hessian, 3x3x3 NMS, octave map, level-drop rule) and `ag_select_keypoints`
(`select_kernel`) on batched pyramids, against the oracle's multi_scale_detector run on the same bits, image by image.

Every case writes B per-image pyramids into one plan's buffer, detects and selects once for the batch into outputs prefilled with a
sentinel, and demands for every image: the oracle's count, its responses bit for bit in the same order, its octave and level indices,
its normalised LAFs within 1e-6, and the sentinel in every row at or beyond the count.  Equal responses are ordered by seq (level slot,
then raster index), the rule the C ABI documents (tests/helpers.py::OracleCandidates; the oracle's torch.topk leaves their order open).
The pyramids come from the GPU blur (bench shapes, odd and tiny shapes, many images) or are built directly (level-drop pyramids,
tiled pyramids whose responses tie), so the stage is tested on inputs no blur would produce as well."""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

import affnet_oracle as O
from helpers import SENTINEL, OracleCandidates, adversarial_pyramid, detector_level_stats, gold, gray_from_rgb, load_weights, synthetic_image

pytestmark = pytest.mark.gpu

DEV = "cuda"
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
MR = 5.192
ISENT = int(SENTINEL)
AG_ERR_CAPACITY = -3
ODD_SHAPES = [(97, 131), (64, 29), (64, 30), (64, 31), (64, 59), (64, 61), (47, 70), (48, 70), (49, 70), (97, 70), (14, 50), (50, 14)]


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


# ---- harness ----------------------------------------------------------------------------------------------------------------------
def plan_sigmas(plan):
    return [[plan.sigma[o][l] for l in range(plan.n_levels)] for o in range(plan.n_octaves)]


def flat_pyramid(plan, pyrs):
    """pyrs[b][o][l] ([1,1,h_o,w_o] or [h_o,w_o]) -> the plan's device buffer: image b of level (o, l) at level_offset[o][l] + b*h_o*w_o."""
    buf = torch.zeros(plan.total_floats, dtype=torch.float32)
    for b, pyr in enumerate(pyrs):
        for o in range(plan.n_octaves):
            n = plan.h[o] * plan.w[o]
            for l in range(plan.n_levels):
                off = plan.level_offset[o][l] + b * n
                buf[off:off + n] = pyr[o][l].reshape(-1)
    return buf.to(DEV)


def gpu_pyramids(L, imgs, nlevels=3, border=5):
    """The GPU blur's pyramid of imgs [B,1,H,W] -> (plan, device buffer, per-image CPU copies pyrs[b][o][l] [1,1,h,w])."""
    from affnet_b200.HandCraftedModules import ScalePyramid
    plan, buf = ScalePyramid(nlevels, 1.6, border).build(imgs.to(DEV).contiguous())
    views, _, _ = ScalePyramid.views(plan, buf)
    pyrs = [[[lv[b:b + 1].cpu() for lv in octave] for octave in views] for b in range(plan.B)]
    return plan, buf, pyrs


class Detector:
    """ag_detect once over a workspace of `cap` candidates per image; select() calls ag_select_keypoints into sentinel-filled outputs."""

    def __init__(self, L, plan, buf, th=0.0, mr=MR, cap=None):
        self.L, self.lib, self.plan = L, L.lib(), plan
        self.cap = cap or max(plan.H * plan.W // 4, 4096)
        self.ws_buf = torch.full((self.lib.ag_detect_ws_bytes(C.byref(plan), self.cap),), 0xFF, dtype=torch.uint8, device=DEV)
        self.ws = L.DetectWs()
        L.check(self.lib.ag_detect_ws_carve(C.byref(plan), self.cap, L.ptr(self.ws_buf), C.byref(self.ws)))
        L.check(self.lib.ag_detect(C.byref(plan), L.ptr(buf), float(th), int(mr), C.byref(self.ws), L.stream_ptr()))

    def cand_counts(self):
        off = self.ws.d_cand_count - self.ws_buf.data_ptr()
        return self.ws_buf[off:off + 4 * self.plan.B].view(torch.int32).cpu()

    def select(self, nf, out_cap=None):
        """-> (rc, (resp [B,out_cap], lafs [B,out_cap,2,3], oct, lvl, count [B])) on the CPU."""
        B, cap = self.plan.B, out_cap or nf
        resp = torch.full((B, cap), SENTINEL, device=DEV)
        lafs = torch.full((B, cap, 2, 3), SENTINEL, device=DEV)
        oc = torch.full((B, cap), ISENT, dtype=torch.int32, device=DEV)
        lv = torch.full((B, cap), ISENT, dtype=torch.int32, device=DEV)
        cnt = torch.full((B,), ISENT, dtype=torch.int32, device=DEV)
        rc = self.lib.ag_select_keypoints(C.byref(self.plan), C.byref(self.ws), int(nf), 1.0, cap, self.L.ptr(resp), self.L.ptr(lafs),
                                          self.L.ptr(oc), self.L.ptr(lv), self.L.ptr(cnt), self.L.stream_ptr())
        torch.cuda.synchronize()
        return rc, tuple(t.cpu() for t in (resp, lafs, oc, lv, cnt))

    def checked_select(self, nf, out_cap=None):
        rc, out = self.select(nf, out_cap)
        self.L.check(rc)
        return out


def assert_image(out, b, exp, tag):
    """Image b of a select output against the expected rows (resp, lafs, oct, lvl); -> number of keypoints compared."""
    resp, lafs, oc, lv, cnt = out
    r, la, po, lo = exp[:4]
    n = r.numel()
    assert int(cnt[b]) == n, (tag, b, int(cnt[b]), n)
    assert torch.equal(resp[b, :n], r), (tag, b)
    assert torch.equal(oc[b, :n].float(), po) and torch.equal(lv[b, :n].float(), lo), (tag, b)
    if n:
        assert (lafs[b, :n] - la).abs().max().item() < 1e-6, (tag, b)
    assert bool((resp[b, n:] == SENTINEL).all()) and bool((lafs[b, n:] == SENTINEL).all()), (tag, b, "rows beyond the count were written")
    assert bool((oc[b, n:] == ISENT).all()) and bool((lv[b, n:] == ISENT).all()), (tag, b, "rows beyond the count were written")
    return n


def cut(exp, k):
    return tuple(t[:k] for t in exp[:4])


def edges(cands):
    """nf values around each image's total before the global top-k: they cross the sorted / unsorted switch."""
    out = {1, 2}
    for c in cands:
        out |= {c.total - 1, c.total, c.total + 1}
    return sorted(v for v in out if 1 <= v <= 16384)


class Tally:
    def __init__(self, name):
        self.name, self.images, self.keypoints, self.calls, self.ties = name, 0, 0, 0, 0

    def report(self, extra=""):
        print("\n%s: %d images, %d select calls, %d keypoints compared with the oracle, %d tie groups cut by the oracle's top-k%s"
              % (self.name, self.images, self.calls, self.keypoints, self.ties, extra))


def check_batch(L, plan, pyrs, nfs, tally, buf=None, th=0.0, mr=MR, tag="", select_all=True):
    """Detect once for the batch; for every nf (and, if select_all, num_features = 0 with room for every candidate) compare every
    image with the oracle.  The oracle's own top-k is rerun for the nf values at the image's edges and the explicit ones."""
    det = Detector(L, plan, flat_pyramid(plan, pyrs) if buf is None else buf, th=th, mr=mr)
    sig = plan_sigmas(plan)
    cands = [OracleCandidates(p, sig, mr, th) for p in pyrs]
    assert int(det.cand_counts().max()) <= det.cap
    calls = [(nf, nf) for nf in (nfs(cands) if callable(nfs) else nfs)]
    if select_all:
        calls.append((0, max([c.total for c in cands] + [1])))
    explicit = set() if callable(nfs) else set(nfs)
    for nf, out_cap in calls:
        out = det.checked_select(nf, out_cap)
        tally.calls += 1
        for b, c in enumerate(cands):
            tally.keypoints += assert_image(out, b, c.select(nf), (tag, nf))
            if nf in explicit or nf <= 0 or nf in (1, 2, c.total - 1, c.total, c.total + 1):
                tally.ties += c.check_against_oracle(nf)
    tally.images += plan.B
    return det, cands


def smooth_noise(shape, g):
    k = torch.ones(1, 1, 5, 5) / 25
    x = torch.rand(1, 1, shape[0] + 4, shape[1] + 4, generator=g) * 255
    return torch.nn.functional.conv2d(x, k)


def mixed_batch(h, w, seed):
    """Two textured images around a constant one (which has no keypoint)."""
    return torch.cat([synthetic_image(h, w, seed), torch.full((1, 1, h, w), 77.0), synthetic_image(h, w, seed + 1)])


# ---- bench shapes, stage isolated ------------------------------------------------------------------------------------------------
def _graf_1024():
    import cv2
    rgb = cv2.resize(gold("graf_full.npz")["rgb"], (1024, 768), interpolation=cv2.INTER_LINEAR)
    return gray_from_rgb(rgb)


@pytest.mark.parametrize("case", ["2x768x1024", "graf1024", "1080x1920", "2160x3840"])
def test_detector_at_bench_shapes_identical_to_oracle(L, case):
    """The GPU pyramid, copied to the host, through the oracle detector: more than 8192 candidates per image, so every select thread
    loops, the radix select takes several passes and the detector's strips and bands have seams (1080p's last octave is 17x30)."""
    if case == "2x768x1024":
        imgs, nf, border = torch.cat([synthetic_image(768, 1024, 1234), synthetic_image(768, 1024, 1235)]), 3000, 5
    elif case == "graf1024":
        imgs, nf, border = _graf_1024(), 3000, 5
    elif case == "1080x1920":
        imgs, nf, border = synthetic_image(1080, 1920, 77), 6000, 5
    else:
        imgs, nf, border = synthetic_image(2160, 3840, 78), 12000, 33
    plan, buf, pyrs = gpu_pyramids(L, imgs, 3, border)
    t = Tally("bench shape %s (%d octaves)" % (case, plan.n_octaves))
    det, cands = check_batch(L, plan, pyrs, [nf, 1, 16384], t, buf=buf, tag=case, select_all=False)
    n_c = det.cand_counts()
    assert int(n_c.min()) > 8192, n_c
    t.report(", raw candidates per image %s" % n_c.tolist())


# ---- odd and tiny shapes, every level count ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("nlevels", [3, 1, 2, 4, 5, 6])
def test_detector_odd_shapes_identical_to_oracle(L, nlevels):
    """Widths around the 30-column strips, heights around the 48-row bands, a side of 14 (one octave); one batch per shape with a
    constant image in the middle.  nlevels != 3 runs the per-level detector (detect_level_kernel, ping-ponged octave maps)."""
    t = Tally("odd shapes, nlevels %d" % nlevels)
    for (h, w) in ODD_SHAPES:
        imgs = mixed_batch(h, w, h * 1000 + w)
        if nlevels == 1:        # the GPU blur refuses sigma 5.54 (35 taps, max 25): the oracle's dense blur builds the pyramid
            plan, buf = L.make_plan(3, h, w, 1, 1.6, 5), None
            pyrs = [O.scale_pyramid(imgs[b:b + 1], 1, 1.6, 5)[0] for b in range(3)]
        else:
            plan, buf, pyrs = gpu_pyramids(L, imgs, nlevels)
        if (h, w) in ((14, 50), (50, 14)):
            assert plan.n_octaves == 1
        check_batch(L, plan, pyrs, edges, t, buf=buf, tag=(h, w, nlevels))
    t.report()


def test_border_at_least_the_image_height_zeroes_every_response(L):
    """int(mrSize) >= h: the reference zeroes the whole NMS map (Utils.py:140-148), so no level is accepted: count 0 (the oracle raises)."""
    plan, buf, pyrs = gpu_pyramids(L, mixed_batch(14, 50, 3), 3)
    det = Detector(L, plan, buf, mr=14.0)
    for c in [OracleCandidates(p, plan_sigmas(plan), 14.0) for p in pyrs]:
        assert c.total == 0
    for nf in (1, 50, 0):
        out = det.checked_select(nf, 64)
        for b in range(plan.B):
            assert_image(out, b, (torch.zeros(0), torch.zeros(0, 2, 3), torch.zeros(0), torch.zeros(0)), ("mr >= h", nf))


# ---- level-drop rule ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nlevels", [3, 1, 2, 4, 5, 6])
def test_level_drop_rule_identical_to_oracle(L, nlevels):
    """Pyramids built directly (tests/helpers.py::adversarial_pyramid) where levels hold 0, 1 or 2 positive maxima, so every accept /
    drop combination of an octave's levels, negative masked responses and wrapping octave maps occur.  Each seed alone (nf at its own
    edges) and stacked 8 to a batch."""
    seeds = range(400) if nlevels == 3 else range(96)
    plan1, plan8 = L.make_plan(1, 40, 40, nlevels, 1.6, 5), L.make_plan(8, 40, 40, nlevels, 1.6, 5)
    assert plan1.n_octaves == 2
    sig = plan_sigmas(plan1)
    pyrs = [adversarial_pyramid(s, nlevels) for s in seeds]
    combos, n_pos = {}, {}
    for p in pyrs:
        st = detector_level_stats(p[0], sig[0], MR)
        combos[tuple(int(s[1]) for s in st)] = combos.get(tuple(int(s[1]) for s in st), 0) + 1
        for s in st:
            n_pos[min(s[0], 3)] = n_pos.get(min(s[0], 3), 0) + 1
    t1, t8 = Tally("level-drop pyramids, nlevels %d, B = 1" % nlevels), Tally("level-drop pyramids, nlevels %d, B = 8" % nlevels)
    empty = 0
    for p in pyrs:
        _, (c,) = check_batch(L, plan1, [p], edges, t1, tag=("adv", nlevels))
        empty += c.total == 0
    for i in range(0, len(pyrs), 8):
        check_batch(L, plan8, pyrs[i:i + 8], edges, t8, tag=("adv8", nlevels, i))
    t1.report("; octave 0 accept combinations %s, levels by n_pos (3 = >= 3) %s, %d images with no accepted level"
              % (sorted(combos.items()), sorted(n_pos.items()), empty))
    t8.report()
    if nlevels == 3:
        assert len(combos) == 8 and empty > 0 and n_pos.get(1, 0) > 0 and n_pos.get(2, 0) > 0


# ---- selection edges and capacity ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sel_case(L):
    """A batch of three 400x560 images (one constant) with a fixed candidate list per image (totals below the 16384-key limit)."""
    plan, buf, pyrs = gpu_pyramids(L, mixed_batch(400, 560, 4321), 3)
    cands = [OracleCandidates(p, plan_sigmas(plan), MR) for p in pyrs]
    return plan, buf, pyrs, cands


def test_selection_edges_identical_to_oracle(L, sel_case):
    """nf around the switch between sorted and unsorted output, and the 16384-key limit of the shared-memory sort (one more is refused
    and nothing is written)."""
    plan, buf, pyrs, cands = sel_case
    det = Detector(L, plan, buf)
    t = Tally("selection edges 3 x 400x560 (totals %s)" % [c.total for c in cands])
    for nf in edges(cands) + [16384]:
        out = det.checked_select(nf)
        t.calls += 1
        for b, c in enumerate(cands):
            t.keypoints += assert_image(out, b, c.select(nf), ("edge", nf))
    rc, out = det.select(16385)
    assert rc == AG_ERR_CAPACITY
    for x in out:
        assert bool((x == SENTINEL).all()) if x.is_floating_point() else bool((x == ISENT).all())
    t.images = plan.B
    t.report()


def test_out_cap_below_the_candidate_total(L, sel_case):
    """out_cap < num_features, and num_features <= 0 or num_features >= total with out_cap < total: the first out_cap keypoints of
    the full answer, in its order (seq order when unsorted), the same on every run."""
    plan, buf, pyrs, cands = sel_case
    det = Detector(L, plan, buf)
    T = max(c.total for c in cands)
    assert T > 2000
    t = Tally("out_cap below the total (totals %s)" % [c.total for c in cands])
    for nf, out_cap in ((0, 100), (-1, 1000), (0, 1), (T, 100), (T + 5, 1500), (3000, 100), (3000, 2999), (T - 1, 37)):
        first = det.checked_select(nf, out_cap)
        again = det.checked_select(nf, out_cap)
        for x, y in zip(first, again):
            assert torch.equal(x, y), (nf, out_cap, "run-dependent output")
        t.calls += 2
        for b, c in enumerate(cands):
            t.keypoints += assert_image(first, b, cut(c.select(nf), out_cap), ("out_cap", nf, out_cap))
    t.images = plan.B
    t.report()


def test_candidate_capacity_at_and_below_the_raw_count(L, sel_case):
    """cand_cap = the largest raw count: the same output; one less: only that image overflows (count -1), the others are unchanged."""
    plan, buf, pyrs, cands = sel_case
    base = Detector(L, plan, buf)
    n_c = base.cand_counts()
    top = int(n_c.max())
    assert int((n_c == top).sum()) == 1, n_c
    big = int(n_c.argmax())
    ref = [base.checked_select(nf) for nf in (1000, 6000)]
    at = Detector(L, plan, buf, cap=top)
    assert torch.equal(at.cand_counts(), n_c)
    for nf, r in zip((1000, 6000), ref):
        for x, y in zip(at.checked_select(nf), r):
            assert torch.equal(x, y), ("cand_cap = max", nf)
    below = Detector(L, plan, buf, cap=top - 1)
    for nf, r in zip((1000, 6000), ref):
        out = below.checked_select(nf)
        assert int(out[4][big]) == -1
        for b in range(plan.B):
            if b != big:
                for x, y in zip(out, r):
                    assert torch.equal(x[b], y[b]), ("cand_cap = max - 1", nf, b)
    print("\ncandidate capacity: raw counts %s, image %d overflows at cand_cap %d" % (n_c.tolist(), big, top - 1))


# ---- ties ------------------------------------------------------------------------------------------------------------------------------
def tiled_pyramid(plan, seed):
    """Every level of every octave tiles one smooth random 32x32 tile, so interior responses repeat bit for bit across tiles."""
    g = torch.Generator().manual_seed(seed)
    pyr = []
    for o in range(plan.n_octaves):
        h, w = plan.h[o], plan.w[o]
        pyr.append([smooth_noise((32, 32), g).repeat(1, 1, h // 32 + 1, w // 32 + 1)[:, :, :h, :w].contiguous() for _ in range(plan.n_levels)])
    return pyr


def test_ties_at_the_cut_follow_seq_order(L):
    plan = L.make_plan(2, 128, 160, 3, 1.6, 5)
    pyrs = [tiled_pyramid(plan, 90 + b) for b in range(2)]
    cands = [OracleCandidates(p, plan_sigmas(plan), MR) for p in pyrs]
    nfs, groups = [], 0
    for c in cands:
        srt = torch.sort(c.resp, descending=True).values
        inside = [i for i in range(1, srt.numel()) if srt[i - 1] == srt[i]]      # nf = i cuts a tie group
        assert len(inside) > 10, len(inside)
        nfs += [inside[0], inside[len(inside) // 2], inside[-1]]
    t = Tally("ties: tiled 2 x 128x160")
    check_batch(L, plan, pyrs, sorted(set(nfs)), t, tag="ties")
    for nf in sorted(set(nfs)):
        for c in cands:
            r = c.select(nf)[0]
            if r.numel() == nf and nf < c.total:
                groups += int(((c.resp == r[-1]).sum() > (r == r[-1]).sum()).item())
    assert groups >= 4, groups
    t.report(", %d (nf, image) cuts fall inside a tie group" % groups)


# ---- many images -------------------------------------------------------------------------------------------------------------------------
def test_many_small_images_identical_to_oracle(L):
    """B = 64 images of 97x131: 512 selection CTAs in 8-CTA clusters."""
    imgs = torch.cat([synthetic_image(97, 131, 500 + b) if b % 9 else torch.full((1, 1, 97, 131), float(b)) for b in range(64)])
    plan, buf, pyrs = gpu_pyramids(L, imgs, 3)
    t = Tally("many images, 64 x 97x131")
    check_batch(L, plan, pyrs, [50, 1], t, buf=buf, tag="B64")
    t.report()


# ---- constructor defaults and thresholds ----------------------------------------------------------------------------------------------
def test_constructor_defaults_and_thresholds(L):
    """ScaleSpaceAffinePatchExtractor() (border 16, mrSize 3.0: NMS border 3, smallest octave 35 px); th mode (th = 5.0, every candidate
    of a full octave set); th > 0 together with a positive num_features."""
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    t = Tally("constructor defaults / thresholds")
    img = synthetic_image(480, 640, 41)
    det = ScaleSpaceAffinePatchExtractor()
    assert det.b == 16 and det.mrSize == 3.0
    for nf in (500, 5000, 1):
        r, la, oc, lv = det.multiScaleDetector(img.to(DEV), nf)
        c = OracleCandidates([[x.cpu() for x in o] for o in det.scale_pyr], det.sigmas, 3.0)
        er, ela, eo, el = c.select(nf)[:4]
        assert torch.equal(r.cpu(), er) and torch.equal(oc.cpu(), eo) and torch.equal(lv.cpu(), el), nf
        assert (la.cpu() - ela).abs().max().item() < 1e-6
        t.keypoints += r.numel(); t.calls += 1; t.ties += c.check_against_oracle(nf)
    det = ScaleSpaceAffinePatchExtractor(mrSize=MR, border=5, th=5.0)
    r, la, oc, lv = det.multiScaleDetector(img.to(DEV), det.num)
    assert det._plan.n_octaves >= 5
    c = OracleCandidates([[x.cpu() for x in o] for o in det.scale_pyr], det.sigmas, MR, th=5.0)
    er, ela, eo, el = c.select(-1)[:4]
    assert r.numel() > 100 and torch.equal(r.cpu(), er) and torch.equal(oc.cpu(), eo) and torch.equal(lv.cpu(), el)
    assert (la.cpu() - ela).abs().max().item() < 1e-6
    t.keypoints += r.numel(); t.calls += 1
    plan, buf, pyrs = gpu_pyramids(L, mixed_batch(200, 328, 8), 3)
    check_batch(L, plan, pyrs, edges, t, buf=buf, th=5.0, tag="th 5")
    t.images += 2
    t.report()


# ---- level counts: limits and the pipeline ------------------------------------------------------------------------------------------
def test_too_many_detection_levels_are_refused(L):
    """nlevels = 6 at 1024x768: 6 octaves x 6 detection levels = 36 slots, above the 32 the candidate key holds."""
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    plan = L.make_plan(1, 768, 1024, 6, 1.6, 5)
    assert plan.n_octaves * (plan.n_levels - 2) == 36
    ws_buf = torch.empty(L.lib().ag_detect_ws_bytes(C.byref(plan), 4096), dtype=torch.uint8, device=DEV)
    with pytest.raises(L.AffnetB200Error, match="32 slots"):
        L.check(L.lib().ag_detect_ws_carve(C.byref(plan), 4096, L.ptr(ws_buf), C.byref(L.DetectWs())))
    with pytest.raises(L.AffnetB200Error, match="32 slots"):
        ScaleSpaceAffinePatchExtractor(mrSize=MR, border=5, nlevels=6).multiScaleDetector(synthetic_image(768, 1024, 1).to(DEV), 100)
    torch.cuda.synchronize()


@pytest.mark.parametrize("nlevels", [2, 4])
def test_pipeline_other_level_counts_equal_single_image_api(L, nlevels):
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    W = load_weights()
    aff, ori, hn = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    aff.load_state_dict(W["affnet"]); ori.load_state_dict(W["orinet"]); hn.load_state_dict(W["hardnet"])
    aff, ori, hn = aff.eval().to(DEV), ori.eval().to(DEV), hn.eval().to(DEV)
    imgs = mixed_batch(200, 328, 61).to(DEV)
    K = 300
    pipe = DetectDescribePipeline(3, 200, 328, aff, hn, ori, num_features=K, nlevels=nlevels, do_ori=True)
    lafs, resp, desc, cnt = [x.clone() for x in pipe.run(imgs)]
    torch.cuda.synchronize()
    det = ScaleSpaceAffinePatchExtractor(mrSize=MR, num_features=K, border=5, num_Baum_iters=1, nlevels=nlevels, AffNet=aff, OriNet=ori)
    for b in range(3):
        dL, r = det(imgs[b:b + 1], do_ori=True)
        n = int(cnt[b])
        assert n == dL.size(0) and (n > 0) == (b != 1), (nlevels, b, n)
        if n:
            d = hn(det.extract_patches_from_pyr(dL, PS=32))
            assert torch.equal(resp[b, :n], r) and torch.equal(lafs[b, :n], dL) and torch.equal(desc[b, :n], d), (nlevels, b)
    print("\npipeline nlevels %d: counts %s" % (nlevels, cnt.tolist()))


# ---- A/B kernel variants ----------------------------------------------------------------------------------------------------------
_SCRIPT = r"""
import sys, torch
sys.path.insert(0, sys.argv[2]); sys.path.insert(0, sys.argv[2] + "/tests"); sys.path.insert(0, sys.argv[2] + "/oracle")
import affnet_b200._lib as L
import test_gpu_detect as T
from helpers import adversarial_pyramid
res = {}
plan, buf, _ = T.gpu_pyramids(L, T.mixed_batch(97, 131, 5), 3)
plan8 = L.make_plan(8, 40, 40, 3, 1.6, 5)
for name, (p, b) in {"odd": (plan, buf), "adv": (plan8, T.flat_pyramid(plan8, [adversarial_pyramid(s) for s in range(8)]))}.items():
    det = T.Detector(L, p, b)
    for nf, cap in ((1, 1), (40, 40), (0, 4096)):
        res["%s_%d" % (name, nf)] = det.checked_select(nf, cap)
torch.save(res, sys.argv[1])
"""


def _run_variant(tmp_path, name, env_extra):
    out = str(tmp_path / (name + ".pt"))
    env = dict(os.environ)
    for k in ("AG_BLUR_NO_TMA", "AG_DETECT_WARP_V1", "AG_DETECT_TILED", "AG_PYR_FUSED"):
        env.pop(k, None)
    env.update(env_extra)
    r = subprocess.run([sys.executable, "-c", _SCRIPT, out, ROOT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return torch.load(out)


def test_detector_variants_agree_with_the_default(tmp_path):
    """The first register formulation (AG_DETECT_WARP_V1) gives the default's bits on the odd-shape and the level-drop batches.  The
    shared-memory tiled detector (AG_DETECT_TILED) makes the same decisions and responses bit for bit, but sums the 27 soft-argmax taps
    one by one where the register kernels add per-row sums, so its LAFs may differ in the last bits: they must stay within the 1e-6 the
    oracle comparison allows."""
    base = _run_variant(tmp_path, "default", {})
    assert int(base["odd_0"][4].max()) > 20 and int(base["adv_0"][4].max()) > 0
    v1 = _run_variant(tmp_path, "v1", {"AG_DETECT_WARP_V1": "1"})
    tiled = _run_variant(tmp_path, "tiled", {"AG_DETECT_TILED": "1"})
    worst = 0.0
    for key in base:
        for i, (x, y, z) in enumerate(zip(base[key], v1[key], tiled[key])):
            assert torch.equal(x, y), ("AG_DETECT_WARP_V1", key, i)
            if i == 1:
                worst = max(worst, (x - z).abs().max().item())
                assert (x - z).abs().max().item() < 1e-6, ("AG_DETECT_TILED", key)
            else:
                assert torch.equal(x, z), ("AG_DETECT_TILED", key, i)
    print("\ndetector variants: AG_DETECT_WARP_V1 bit-identical; AG_DETECT_TILED identical but for LAFs, max |dLAF| %.2e" % worst)
