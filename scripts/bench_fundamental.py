"""Device fundamental-matrix RANSAC (ReprojectionStuff.find_fundamental_pairs, inl_th = 0.5) against today's practice (counts and
tentatives to the host, then a Python loop of cv2.findFundamentalMat(FM_RANSAC, 0.5, 0.99, 50000) per pair).  Workloads: the 8
two-plane pairs of tests/test_gpu_fundamental.py (one B = 16 pipeline batch, AffNet + histogram orientation, K = 2000); the 15
consecutive and 240 ordered pairs of scripts/bench_matching.py's workload (16 x 1024x768 synthetic images, K = 2000, AffNet + OriNet,
HardNet), whose unrelated images leave 1-15 tentatives per pair; and constructed n = 1000 pairs with 40 % outliers
(tests/fundamental_cases.scene) at P = 1, 132 and 1024, the cv2 loop for P = 1 only (one such pair took cv2 0.26-0.53 s).  Device:
CUDA-event time of a CUDA-graph replay of the call alone (median of --steps after --warmup).  Host loop: host clock from before the count read to the end of the loop (median).  Also records
samples and inliers per pair, and the card's name and power limit, read in the same run.

    python scripts/bench_fundamental.py [--steps 20] [--warmup 5] [--out FILE.json]

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
from bench_verify import graph_ms  # noqa: E402

TH = 0.5


def cv2_loop(cv2, lafs1, lafs2, tent, ntent, pl):
    """Today's practice: counts and tentatives to the host, then cv2.findFundamentalMat per pair -> inlier counts."""
    nt = ntent.tolist()
    out = []
    for p, (i, j) in enumerate(pl):
        n = nt[p]
        if n < 8:   # FM_RANSAC needs 8 points (cv2 solves 7 with FM_7POINT only); the device call also samples pairs of 7
            out.append(0)
            continue
        t = tent[p, :n].long()
        a = lafs1[i, t[:, 0], :, 2].cpu().numpy()
        b = lafs2[j, t[:, 1], :, 2].cpu().numpy()
        F, m = cv2.findFundamentalMat(a, b, cv2.FM_RANSAC, TH, 0.99, 50000)
        out.append(0 if m is None else int(m.sum()))
    return out


def measure(lafs1, lafs2, tent, ntent, pl, steps, warmup, cv2, cv2_reps=None, host=True):
    from affnet_b200.ReprojectionStuff import find_fundamental_pairs, find_homography_pairs
    pairs = torch.tensor(pl, dtype=torch.int32, device="cuda")
    ft, (F, inl, ninl, iters) = graph_ms(lambda: find_fundamental_pairs(lafs1, tent, ntent, lafs2, pairs), steps, warmup)
    _, (H, hinl, hninl, hiters) = graph_ms(lambda: find_homography_pairs(lafs1, tent, ntent, lafs2, pairs), 1, 0)
    torch.cuda.synchronize()
    r = dict(pairs=len(pl), tentatives=ntent.tolist(), fundamental_graph_ms=ft, fundamental_inliers=ninl.tolist(),
             fundamental_samples=iters.tolist(), homography_inliers=hninl.tolist())
    if cv2 is None:
        r["host_baseline"] = "skipped: cv2 is not importable"
    elif not host:
        r["host_baseline"] = "not run: the P = 1 row gives the cv2 cost of one such pair"
    else:
        reps = cv2_reps or max(3, steps // 4)
        cv2_loop(cv2, lafs1, lafs2, tent, ntent, pl)
        ms = []
        for _ in range(reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            inl_cv = cv2_loop(cv2, lafs1, lafs2, tent, ntent, pl)
            ms.append((time.perf_counter() - t0) * 1e3)
        ms.sort()
        r["host_cv2_loop_ms"] = dict(median=ms[len(ms) // 2], min=ms[0], max=ms[-1], reps=reps)
        r["cv2_inliers"] = inl_cv
        r["speedup_cv2_loop_over_device"] = ms[len(ms) // 2] / ft["median"]
    print("P=%4d  device %8.3f ms  cv2 loop %s ms" % (len(pl), ft["median"],
          "%.3f" % r["host_cv2_loop_ms"]["median"] if "host_cv2_loop_ms" in r else "-"), file=sys.stderr)
    return r


def constructed(P, n=1000, cap=1000):
    """P pairs of seeded 3D scenes (n = 1000, 40 % outliers, 0.3 px noise) as LAF sets and tentatives."""
    import fundamental_cases as FC
    l1, l2 = torch.zeros(P, cap, 2, 3), torch.zeros(P, cap, 2, 3)
    for p in range(P):
        pts, _, _ = FC.scene(3000 + p, n)
        q = torch.from_numpy(pts)
        l1[p, :n, 0, 2], l1[p, :n, 1, 2], l2[p, :n, 0, 2], l2[p, :n, 1, 2] = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    rows = torch.arange(n, dtype=torch.int32)
    tent = torch.stack([rows, rows], 1)[None].repeat(P, 1, 1).contiguous()
    ntent = torch.full((P,), n, dtype=torch.int32)
    return l1.cuda(), l2.cuda(), tent.cuda(), ntent.cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fundamental.py needs a CUDA device")
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
    from test_gpu_fundamental import two_plane_pairs
    W = load_weights()
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    a, o, h = a.eval().cuda(), o.eval().cuda(), h.eval().cuda()
    res = dict(card=card(), steps=args.steps, warmup=args.warmup, inl_th=TH, cv2=None if cv2 is None else cv2.__version__, workloads={})
    B, Hh, Ww, K = 16, 768, 1024, 2000

    imgs, _ = two_plane_pairs(Hh, Ww)
    pipe = DetectDescribePipeline(16, Hh, Ww, a, h, None, num_features=K, do_ori=True)
    lafs, _, desc, cnt = pipe.run(imgs.cuda())
    pipe.check()
    pl = [(2 * k, 2 * k + 1) for k in range(8)]
    tent, ntent, _, _ = match_snn_pairs(desc, cnt, pairs=torch.tensor(pl, device="cuda"))
    res["workloads"]["8 two-plane pairs 1024x768, K = 2000, AffNet + histogram"] = measure(lafs, lafs, tent, ntent, pl, args.steps,
                                                                                             args.warmup, cv2)
    del pipe
    torch.cuda.empty_cache()

    pipe = DetectDescribePipeline(B, Hh, Ww, a, h, o, num_features=K)
    lafs, _, desc, cnt = pipe.run(torch.cat([synthetic_image(Hh, Ww, 1234 + i) for i in range(B)]).cuda())
    pipe.check()
    lafs, cnt = lafs.clone(), cnt.clone()
    for pname, pl in (("15 consecutive pairs", [(i, i + 1) for i in range(15)]),
                      ("240 ordered pairs", [(i, j) for i in range(16) for j in range(16) if i != j])):
        tent, ntent, _, _ = match_snn_pairs(desc, cnt, pairs=torch.tensor(pl, device="cuda"))
        res["workloads"]["16 x 1024x768 unrelated images, K = 2000, " + pname] = measure(lafs, lafs, tent, ntent, pl, args.steps,
                                                                                         args.warmup, cv2)
    del pipe
    torch.cuda.empty_cache()

    for P in (1, 132, 1024):
        l1, l2, tent, ntent = constructed(P)
        pl = [(p, p) for p in range(P)]
        res["workloads"]["constructed n = 1000, 40 %% outliers, P = %d" % P] = measure(l1, l2, tent, ntent, pl, args.steps, args.warmup,
                                                                                      cv2, cv2_reps=3, host=P == 1)
    res["card"]["after"] = card()["nvidia_smi"]
    doc = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(doc + "\n")
    print(doc)


if __name__ == "__main__":
    main()
