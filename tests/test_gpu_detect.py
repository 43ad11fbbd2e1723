"""GPU tests (-m gpu) of the detector stage alone: `ag_detect` (Hessian, 3x3x3 NMS, octave map, level-drop rule) and `ag_select_keypoints`
(`select_kernel`) on batched pyramids, against the oracle's multi_scale_detector run on the same bits, image by image.

Every case writes B per-image pyramids into one plan's buffer, detects and selects once for the batch into outputs prefilled with a
sentinel, and demands for every image: the oracle's count, its responses bit for bit in the same order, its octave and level indices,
its normalised LAFs bit for bit as the soft-argmax restatement of the kernel's summation order computes them (tests/detect_restated.py),
and the sentinel in every row at or beyond the count.  Equal responses are ordered by seq (level slot,
then raster index), the rule the C ABI documents (tests/helpers.py::OracleCandidates; the oracle's torch.topk leaves their order open).
The pyramids come from the GPU blur (bench shapes, odd and tiny shapes, many images) or are built directly (level-drop pyramids,
tiled pyramids whose responses tie), so the stage is tested on inputs no blur would produce as well."""
import ctypes as C

import numpy as np
import pytest
import torch

import affnet_oracle as O
from detect_restated import Restated, bits
from helpers import (SENTINEL, Detector, OracleCandidates, adversarial_pyramid, detector_level_stats, flat_pyramid, gold, gpu_pyramids,
                     gray_from_rgb, load_weights, mixed_batch, plan_sigmas, synthetic_image)

pytestmark = pytest.mark.gpu

DEV = "cuda"
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
def order_of(plan):
    """The soft-argmax order of the default build: the register kernel at 3 detection levels, detect_level_kernel otherwise."""
    return "rows" if plan.n_levels - 2 == 3 else "taps"


def restate(cands, order):
    return [Restated(c.pyr, c.sigmas, c.seq, order, th=c.th) for c in cands]


def expected(c, R, nf):
    """c.select(nf) with the LAFs the kernel writes (R: c's restated rows, tests/detect_restated.py) in place of the oracle's."""
    idx = torch.from_numpy(np.ascontiguousarray(c.order(nf)[0])).long()
    return c.resp[idx], R.lafs32[idx], c.oct[idx], c.lvl[idx]


def assert_image(out, b, exp, tag):
    """Image b of a select output against the expected rows (resp, lafs, oct, lvl); -> number of keypoints compared."""
    resp, lafs, oc, lv, cnt = out
    r, la, po, lo = exp[:4]
    n = r.numel()
    assert int(cnt[b]) == n, (tag, b, int(cnt[b]), n)
    assert torch.equal(resp[b, :n], r), (tag, b)
    assert torch.equal(oc[b, :n].float(), po) and torch.equal(lv[b, :n].float(), lo), (tag, b)
    assert torch.equal(bits(lafs[b, :n]), bits(la)), (tag, b, "LAFs differ from the restated soft-argmax")
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
    Rs = restate(cands, order_of(plan))
    assert int(det.cand_counts().max()) <= det.cap
    calls = [(nf, nf) for nf in (nfs(cands) if callable(nfs) else nfs)]
    if select_all:
        calls.append((0, max([c.total for c in cands] + [1])))
    explicit = set() if callable(nfs) else set(nfs)
    for nf, out_cap in calls:
        out = det.checked_select(nf, out_cap)
        tally.calls += 1
        for b, (c, R) in enumerate(zip(cands, Rs)):
            tally.keypoints += assert_image(out, b, expected(c, R, nf), (tag, nf))
            if nf in explicit or nf <= 0 or nf in (1, 2, c.total - 1, c.total, c.total + 1):
                tally.ties += c.check_against_oracle(nf)
    tally.images += plan.B
    return det, cands, Rs


def smooth_noise(shape, g):
    k = torch.ones(1, 1, 5, 5) / 25
    x = torch.rand(1, 1, shape[0] + 4, shape[1] + 4, generator=g) * 255
    return torch.nn.functional.conv2d(x, k)


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
    det, cands, _ = check_batch(L, plan, pyrs, [nf, 1, 16384], t, buf=buf, tag=case, select_all=False)
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
        _, (c,), _ = check_batch(L, plan1, [p], edges, t1, tag=("adv", nlevels))
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
    return plan, buf, pyrs, cands, restate(cands, "rows")


def test_selection_edges_identical_to_oracle(L, sel_case):
    """nf around the switch between sorted and unsorted output, and the 16384-key limit of the shared-memory sort (one more is refused
    and nothing is written)."""
    plan, buf, pyrs, cands, Rs = sel_case
    det = Detector(L, plan, buf)
    t = Tally("selection edges 3 x 400x560 (totals %s)" % [c.total for c in cands])
    for nf in edges(cands) + [16384]:
        out = det.checked_select(nf)
        t.calls += 1
        for b, c in enumerate(cands):
            t.keypoints += assert_image(out, b, expected(c, Rs[b], nf), ("edge", nf))
    rc, out = det.select(16385)
    assert rc == AG_ERR_CAPACITY
    for x in out:
        assert bool((x == SENTINEL).all()) if x.is_floating_point() else bool((x == ISENT).all())
    t.images = plan.B
    t.report()


def test_out_cap_below_the_candidate_total(L, sel_case):
    """out_cap < num_features, and num_features <= 0 or num_features >= total with out_cap < total: the first out_cap keypoints of
    the full answer, in its order (seq order when unsorted), the same on every run."""
    plan, buf, pyrs, cands, Rs = sel_case
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
            t.keypoints += assert_image(first, b, cut(expected(c, Rs[b], nf), out_cap), ("out_cap", nf, out_cap))
    t.images = plan.B
    t.report()


def test_candidate_capacity_at_and_below_the_raw_count(L, sel_case):
    """cand_cap = the largest raw count: the same output; one less: only that image overflows (count -1), the others are unchanged."""
    plan, buf, pyrs, cands, _ = sel_case
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
        er, ela, eo, el = expected(c, restate([c], "rows")[0], nf)
        assert torch.equal(r.cpu(), er) and torch.equal(oc.cpu(), eo) and torch.equal(lv.cpu(), el), nf
        assert torch.equal(bits(la.cpu()), bits(ela)), nf
        t.keypoints += r.numel(); t.calls += 1; t.ties += c.check_against_oracle(nf)
    det = ScaleSpaceAffinePatchExtractor(mrSize=MR, border=5, th=5.0)
    r, la, oc, lv = det.multiScaleDetector(img.to(DEV), det.num)
    assert det._plan.n_octaves >= 5
    c = OracleCandidates([[x.cpu() for x in o] for o in det.scale_pyr], det.sigmas, MR, th=5.0)
    er, ela, eo, el = expected(c, restate([c], "rows")[0], -1)
    assert r.numel() > 100 and torch.equal(r.cpu(), er) and torch.equal(oc.cpu(), eo) and torch.equal(lv.cpu(), el)
    assert torch.equal(bits(la.cpu()), bits(ela))
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
