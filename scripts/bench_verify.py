"""Device verification of the batched matcher's tentatives (ReprojectionStuff.find_homography_pairs / gt_correspondences_pairs)
against today's practice (the counts read to the host, then a Python loop of cv2.findHomography(RANSAC, 2.0) per pair).  Workloads of
scripts/bench_matching.py: 16 x 1024x768 synthetic images at K = 2000 (AffNet + OriNet, HardNet), the 15 consecutive pairs and the 240
ordered pairs i != j; plus the 8 warped pairs of tests/test_gpu_verify.py (AffNet + histogram orientation, one B = 16 batch), where the
true homographies are known.  Device: CUDA-event time of a CUDA-graph replay of each call alone (median of --steps after --warmup).
Host loop: host clock from before the count read to the end of the loop (median).  Also records iterations and inliers per pair, and the
card's name and power limit, read in the same run.

    python scripts/bench_verify.py [--steps 20] [--warmup 5] [--out FILE.json]

Needs an H100 (there is no CPU path); prints one JSON document.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_matching import card  # noqa: E402


def graph_ms(fn, steps, warmup):
    """Median / min / max CUDA-event time of a CUDA-graph replay of fn()."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    for _ in range(warmup):
        g.replay()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    ms.sort()
    return dict(median=ms[len(ms) // 2], min=ms[0], max=ms[-1]), out


def cv2_loop(cv2, lafs, tent, ntent, pl):
    """Today's practice: counts and tentatives to the host, then cv2.findHomography per pair -> inlier counts."""
    nt = ntent.tolist()
    out = []
    for p, (i, j) in enumerate(pl):
        n = nt[p]
        if n < 4:
            out.append(0)
            continue
        t = tent[p, :n].long()
        a = lafs[i, t[:, 0], :, 2].cpu().numpy()
        b = lafs[j, t[:, 1], :, 2].cpu().numpy()
        H, m = cv2.findHomography(a, b, cv2.RANSAC, 2.0, maxIters=50000, confidence=0.99)
        out.append(0 if m is None else int(m.sum()))
    return out


def measure(lafs, tent, ntent, pl, Hgt, steps, warmup, cv2):
    from affnet_b200.ReprojectionStuff import find_homography_pairs, gt_correspondences_pairs
    pairs = torch.tensor(pl, dtype=torch.int32, device="cuda")
    Ht = Hgt if Hgt is not None else torch.eye(3, device="cuda").expand(len(pl), 3, 3).contiguous()
    rt, (H, inl, ninl, iters) = graph_ms(lambda: find_homography_pairs(lafs, tent, ntent, pairs=pairs), steps, warmup)
    gt, (true, ntrue, _, _) = graph_ms(lambda: gt_correspondences_pairs(lafs, tent, ntent, Ht, pairs=pairs), steps, warmup)
    torch.cuda.synchronize()
    r = dict(pairs=len(pl), tentatives=ntent.tolist(), ransac_graph_ms=rt, gt_graph_ms=gt, ransac_inliers=ninl.tolist(),
             ransac_iterations=iters.tolist())
    if Hgt is not None:
        from verify_cases import corner_error
        r["gt_true"] = ntrue.tolist()
        r["corner_error_px"] = [corner_error(H[p].cpu().numpy(), Hgt[p].cpu().numpy().astype(np.float64)) for p in range(len(pl))]
    if cv2 is None:
        r["host_baseline"] = "skipped: cv2 is not importable"
    else:
        for _ in range(max(1, warmup // 2)):
            cv2_loop(cv2, lafs, tent, ntent, pl)
        ms = []
        for _ in range(max(3, steps // 4)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            inl_cv = cv2_loop(cv2, lafs, tent, ntent, pl)
            ms.append((time.perf_counter() - t0) * 1e3)
        ms.sort()
        r["host_cv2_loop_ms"] = dict(median=ms[len(ms) // 2], min=ms[0], max=ms[-1])
        r["cv2_inliers"] = inl_cv
        r["speedup_cv2_loop_over_device_ransac"] = ms[len(ms) // 2] / rt["median"]
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_verify.py needs a CUDA device")
    try:
        import cv2
        cv2.setNumThreads(1)
    except ImportError:
        cv2 = None
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from helpers import load_weights, synthetic_image
    from test_gpu_verify import warp
    from verify_cases import random_homography
    W = load_weights()
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    a, o, h = a.eval().cuda(), o.eval().cuda(), h.eval().cuda()
    res = dict(card=card(), steps=args.steps, warmup=args.warmup, cv2=None if cv2 is None else cv2.__version__, workloads={})

    B, Hh, Ww, K = 16, 768, 1024, 2000
    pipe = DetectDescribePipeline(B, Hh, Ww, a, h, o, num_features=K)
    lafs, _, desc, cnt = pipe.run(torch.cat([synthetic_image(Hh, Ww, 1234 + i) for i in range(B)]).cuda())
    pipe.check()
    lafs, cnt = lafs.clone(), cnt.clone()
    for pname, pl in (("15 consecutive pairs", [(i, i + 1) for i in range(15)]),
                      ("240 ordered pairs", [(i, j) for i in range(16) for j in range(16) if i != j])):
        tent, ntent, _, _ = match_snn_pairs(desc, cnt, pairs=torch.tensor(pl, device="cuda"))
        r = measure(lafs, tent, ntent, pl, None, args.steps, args.warmup, cv2)
        res["workloads"]["16 x 1024x768, K = 2000, " + pname] = r
        print("%-22s ransac %7.3f ms  gt %7.3f ms  cv2 loop %s ms" % (pname, r["ransac_graph_ms"]["median"], r["gt_graph_ms"]["median"],
              "%.3f" % r["host_cv2_loop_ms"]["median"] if cv2 else "-"), file=sys.stderr)
    del pipe
    torch.cuda.empty_cache()

    Hs = [random_homography(500 + k, Hh, Ww) for k in range(8)]
    imgs = []
    for k in range(8):
        x = synthetic_image(Hh, Ww, 900 + k)
        imgs += [x, warp(x, Hs[k])]
    pipe = DetectDescribePipeline(16, Hh, Ww, a, h, None, num_features=K, do_ori=True)
    lafs, _, desc, cnt = pipe.run(torch.cat(imgs).cuda())
    pipe.check()
    pl = [(2 * k, 2 * k + 1) for k in range(8)]
    tent, ntent, _, _ = match_snn_pairs(desc, cnt, pairs=torch.tensor(pl, device="cuda"))
    Hgt = torch.from_numpy(np.stack(Hs).astype(np.float32)).cuda()
    r = measure(lafs, tent, ntent, pl, Hgt, args.steps, args.warmup, cv2)
    res["workloads"]["8 warped pairs 1024x768, K = 2000, AffNet + histogram"] = r
    print("%-22s ransac %7.3f ms  gt %7.3f ms  cv2 loop %s ms" % ("8 warped pairs", r["ransac_graph_ms"]["median"], r["gt_graph_ms"]["median"],
          "%.3f" % r["host_cv2_loop_ms"]["median"] if cv2 else "-"), file=sys.stderr)
    res["card"]["after"] = card()["nvidia_smi"]
    doc = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(doc + "\n")
    print(doc)


if __name__ == "__main__":
    main()
