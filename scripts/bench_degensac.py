"""Device DEGENSAC (ReprojectionStuff.find_fundamental_pairs(degensac=True), inl_th = 0.5) against the plain device RANSAC
(degensac=False) and a host loop of cv2.findFundamentalMat(USAC_DEFAULT, 0.5, 0.99, 50000).  Workloads: those of
scripts/bench_fundamental.py (the 8 two-plane pairs, the 15 consecutive and 240 ordered pairs of 16 unrelated images, constructed
n = 1000 scenes at P = 1, 132, 1024), plus dominant-plane pairs (tests/degensac_cases.dominant_plane: n = 600, 30 % outliers,
15 % of the true matches off the plane) at P = 1, 132 and 1024.  Device: CUDA-event time of a CUDA-graph replay of the call alone
(median of --steps after --warmup), plain and DEGENSAC alternated --rounds times in the same process.  Host loop (P = 1 only): host
clock around the loop (median).  Also records inliers and samples per pair (and, for dominant-plane pairs, the fraction of the
off-plane true matches found), and the card's name and power limit, read in the same run.

    python scripts/bench_degensac.py [--steps 20] [--warmup 5] [--rounds 2] [--out FILE.json]

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

from bench_fundamental import constructed  # noqa: E402
from bench_matching import card  # noqa: E402
from bench_verify import graph_ms  # noqa: E402

TH = 0.5


def cv2_usac_loop(cv2, lafs1, lafs2, tent, ntent, pl):
    """Counts and tentatives to the host, then cv2.findFundamentalMat(USAC_DEFAULT) per pair -> inlier masks (None below 8 rows)."""
    nt = ntent.tolist()
    out = []
    for p, (i, j) in enumerate(pl):
        n = nt[p]
        if n < 8:
            out.append(None)
            continue
        t = tent[p, :n].long()
        a = lafs1[i, t[:, 0], :, 2].cpu().numpy()
        b = lafs2[j, t[:, 1], :, 2].cpu().numpy()
        F, m = cv2.findFundamentalMat(a, b, cv2.USAC_DEFAULT, TH, 0.99, 50000)
        out.append(None if m is None else m.ravel().astype(bool))
    return out


def measure(lafs1, lafs2, tent, ntent, pl, args, cv2, host, offp=None):
    from affnet_b200.ReprojectionStuff import find_fundamental_pairs
    pairs = torch.tensor(pl, dtype=torch.int32, device="cuda")
    times = dict(plain=[], degensac=[])
    outs = {}
    for _ in range(args.rounds):
        for mode in ("plain", "degensac"):
            t, o = graph_ms(lambda: find_fundamental_pairs(lafs1, tent, ntent, lafs2, pairs, degensac=mode == "degensac"), args.steps,
                            args.warmup)
            times[mode].append(t)
            outs[mode] = o
    torch.cuda.synchronize()
    r = dict(pairs=len(pl), tentatives=ntent.tolist())
    for mode in ("plain", "degensac"):
        F, inl, ninl, iters = outs[mode]
        r[mode] = dict(graph_ms=times[mode], median_ms=sorted(t["median"] for t in times[mode]), inliers=ninl.tolist(),
                       samples=iters.tolist())
        if offp is not None:
            r[mode]["off_plane_found"] = [float(inl[p, :len(o)].cpu().numpy().astype(bool)[o].mean()) for p, o in enumerate(offp)]
    if cv2 is None:
        r["host_baseline"] = "skipped: cv2 is not importable"
    elif not host:
        r["host_baseline"] = "not run: the P = 1 row gives the cv2 cost of one such pair"
    else:
        cv2_usac_loop(cv2, lafs1, lafs2, tent, ntent, pl)
        ms = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            masks = cv2_usac_loop(cv2, lafs1, lafs2, tent, ntent, pl)
            ms.append((time.perf_counter() - t0) * 1e3)
        ms.sort()
        r["host_cv2_usac_loop_ms"] = dict(median=ms[1], min=ms[0], max=ms[-1], reps=3)
        r["cv2_usac_inliers"] = [0 if m is None else int(m.sum()) for m in masks]
        if offp is not None:
            r["cv2_usac_off_plane_found"] = [None if m is None else float(m[o].mean()) for m, o in zip(masks, offp)]
    print("P=%4d  plain %8.3f ms  degensac %8.3f ms" % (len(pl), times["plain"][-1]["median"], times["degensac"][-1]["median"]),
          file=sys.stderr)
    return r


def dominant(P, n=600):
    """P dominant-plane pairs (seeds 0..P-1) as LAF sets and tentatives, and the off-plane true matches of each."""
    import degensac_cases as DC
    l1, l2 = torch.zeros(P, n, 2, 3), torch.zeros(P, n, 2, 3)
    offp = []
    for p in range(P):
        pts, out, _, off = DC.dominant_plane(p, n)
        q = torch.from_numpy(pts)
        l1[p, :, 0, 2], l1[p, :, 1, 2], l2[p, :, 0, 2], l2[p, :, 1, 2] = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        offp.append(~out & off)
    rows = torch.arange(n, dtype=torch.int32)
    tent = torch.stack([rows, rows], 1)[None].repeat(P, 1, 1).contiguous()
    ntent = torch.full((P,), n, dtype=torch.int32)
    return l1.cuda(), l2.cuda(), tent.cuda(), ntent.cuda(), offp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_degensac.py needs a CUDA device")
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
    res = dict(card=card(), steps=args.steps, warmup=args.warmup, rounds=args.rounds, inl_th=TH,
               cv2=None if cv2 is None else cv2.__version__, workloads={})
    B, Hh, Ww, K = 16, 768, 1024, 2000

    imgs, _ = two_plane_pairs(Hh, Ww)
    pipe = DetectDescribePipeline(16, Hh, Ww, a, h, None, num_features=K, do_ori=True)
    lafs, _, desc, cnt = pipe.run(imgs.cuda())
    pipe.check()
    pl = [(2 * k, 2 * k + 1) for k in range(8)]
    tent, ntent, _, _ = match_snn_pairs(desc, cnt, pairs=torch.tensor(pl, device="cuda"))
    res["workloads"]["8 two-plane pairs 1024x768, K = 2000, AffNet + histogram"] = measure(lafs, lafs, tent, ntent, pl, args, cv2, False)
    del pipe
    torch.cuda.empty_cache()

    pipe = DetectDescribePipeline(B, Hh, Ww, a, h, o, num_features=K)
    lafs, _, desc, cnt = pipe.run(torch.cat([synthetic_image(Hh, Ww, 1234 + i) for i in range(B)]).cuda())
    pipe.check()
    lafs, cnt = lafs.clone(), cnt.clone()
    for pname, pl in (("15 consecutive pairs", [(i, i + 1) for i in range(15)]),
                      ("240 ordered pairs", [(i, j) for i in range(16) for j in range(16) if i != j])):
        tent, ntent, _, _ = match_snn_pairs(desc, cnt, pairs=torch.tensor(pl, device="cuda"))
        res["workloads"]["16 x 1024x768 unrelated images, K = 2000, " + pname] = measure(lafs, lafs, tent, ntent, pl, args, cv2, False)
    del pipe
    torch.cuda.empty_cache()

    for P in (1, 132, 1024):
        l1, l2, tent, ntent = constructed(P)
        pl = [(p, p) for p in range(P)]
        res["workloads"]["constructed n = 1000, 40 %% outliers, P = %d" % P] = measure(l1, l2, tent, ntent, pl, args, cv2, P == 1)
    for P in (1, 132, 1024):
        l1, l2, tent, ntent, offp = dominant(P)
        pl = [(p, p) for p in range(P)]
        r = measure(l1, l2, tent, ntent, pl, args, cv2, P == 1, offp)
        for mode in ("plain", "degensac"):
            f = np.array(r[mode]["off_plane_found"])
            r[mode]["off_plane_found_summary"] = dict(mean=float(f.mean()), min=float(f.min()), share_at_least_0_8=float((f >= 0.8).mean()))
        res["workloads"]["dominant plane n = 600, 30 %% outliers, 15 %% off-plane, P = %d" % P] = r
    res["card"]["after"] = card()["nvidia_smi"]
    doc = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(doc + "\n")
    print(doc)


if __name__ == "__main__":
    main()
