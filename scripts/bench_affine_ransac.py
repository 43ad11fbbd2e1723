"""Device homography RANSAC from two affine correspondences (ReprojectionStuff.find_homography_pairs(affine=True)) against the 4-point
device RANSAC (affine=False), both at inl_th = 2 px.  Workloads: the 8 warped pipeline pairs of tests/test_gpu_ac_ransac.py, the 240
ordered pairs of 16 unrelated images (no true matches: the largest chance inlier count of each method), and constructed n = 1000 scenes
with frames (tests/affine_cases.scene, 5 % frame outliers) at 40 %, 70 % and 85 % outliers for P = 1, 132 and 1024.  Time: CUDA-event
time of a CUDA-graph replay of the call alone (median of --steps after --warmup), 4-point and 2-AC alternated --rounds times in the same
process.  Also records inliers and samples per pair, and the distribution of the frame distance D = |A1^-1 J A2 - I|_F^2 under the
true H over the GT-true tentatives (6 px) of the warped pairs and graf 1->6, from which find_homography_pairs' default laf_th is chosen:
the smallest of {0.5, 1, 2, 4} that keeps at least 95 % of them.  The card's name and power limit are read in the same run.

    python scripts/bench_affine_ransac.py [--steps 10] [--warmup 3] [--rounds 2] [--out FILE.json]

Needs an H100 (there is no CPU path); prints one JSON document.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_matching import card  # noqa: E402
from bench_verify import graph_ms  # noqa: E402

CANDIDATES = (0.5, 1.0, 2.0, 4.0)


def measure(lafs1, lafs2, tent, ntent, pl, args):
    from affnet_b200.ReprojectionStuff import find_homography_pairs
    pairs = torch.tensor(pl, dtype=torch.int32, device="cuda")
    times = {"4-point": [], "2-AC": []}
    outs = {}
    for _ in range(args.rounds):
        for mode in ("4-point", "2-AC"):
            t, o = graph_ms(lambda: find_homography_pairs(lafs1, tent, ntent, lafs2, pairs, affine=mode == "2-AC"), args.steps, args.warmup)
            times[mode].append(t)
            outs[mode] = o
    torch.cuda.synchronize()
    per_pair = len(pl) <= 240        # per-pair lists up to 240 pairs; larger workloads keep the totals
    r = dict(pairs=len(pl), tentatives=ntent.tolist() if per_pair else "n = %d each" % int(ntent[0]))
    for mode in ("4-point", "2-AC"):
        _, _, ninl, iters = outs[mode]
        r[mode] = dict(graph_ms=times[mode], median_ms=sorted(t["median"] for t in times[mode]), max_inliers=int(ninl.max()),
                       max_samples=int(iters.max()), total_inliers=int(ninl.clamp(min=0).sum()), total_samples=int(iters.clamp(min=0).sum()))
        if per_pair:
            r[mode].update(inliers=ninl.tolist(), samples=iters.tolist())
    print("P=%4d  4-point %8.3f ms  2-AC %8.3f ms" % (len(pl), times["4-point"][-1]["median"], times["2-AC"][-1]["median"]), file=sys.stderr)
    return r


def constructed(P, outliers, n=1000):
    """P constructed pairs (seeds 4000 + p) with frames as LAF sets and tentatives."""
    import affine_cases as AC
    l1, l2 = np.zeros((P, n, 2, 3), np.float32), np.zeros((P, n, 2, 3), np.float32)
    for p in range(P):
        l1[p], l2[p], _, _ = AC.scene(4000 + p, n, outliers=outliers, frame_outliers=0.05)
    rows = torch.arange(n, dtype=torch.int32)
    tent = torch.stack([rows, rows], 1)[None].repeat(P, 1, 1).contiguous()
    ntent = torch.full((P,), n, dtype=torch.int32)
    return torch.from_numpy(l1).cuda(), torch.from_numpy(l2).cuda(), tent.cuda(), ntent.cuda()


def true_frame_distances(lafs, tent, ntent, pairs, Hs, px=6.0):
    """D under the true H of each pair's GT-true tentatives (gt_correspondences_pairs at px) -> list of arrays."""
    import oracle_ac_ransac as A
    from affnet_b200.ReprojectionStuff import gt_correspondences_pairs
    Ht = torch.from_numpy(np.stack(Hs).astype(np.float32)).cuda()
    true, ntrue, _, _ = gt_correspondences_pairs(lafs, tent, ntent, Ht, pairs=pairs, dist_threshold=px)
    out = []
    for p in range(pairs.size(0)):
        i, j = (int(v) for v in pairs[p])
        t = tent[p, true[p, :int(ntrue[p])].long()].long()
        ac = A.ac_rows(lafs[i, t[:, 0]].cpu().numpy(), lafs[j, t[:, 1]].cpu().numpy()).astype(np.float64)
        D, ok = A.frame_distance(np.asarray(Hs[p], np.float32).astype(np.float64).reshape(9), ac)
        out.append(np.where(ok[0], D[0], np.inf))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_affine_ransac.py needs a CUDA device")
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.ReprojectionStuff import AFFINE_LAF_TH
    from helpers import load_weights, synthetic_image
    from test_gpu_ac_ransac import graf_pair, warped_pairs
    W = load_weights()
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    a, o, h = a.eval().cuda(), o.eval().cuda(), h.eval().cuda()
    res = dict(card=card(), steps=args.steps, warmup=args.warmup, rounds=args.rounds, inl_th=2.0, laf_th=AFFINE_LAF_TH, workloads={})

    # the frame distance of GT-true tentatives under the true H, and the default it gives
    lafs, tent, ntent, pairs, Hs, _, _ = warped_pairs((a, o, h))
    Dw = true_frame_distances(lafs, tent, ntent, pairs, Hs)
    res["workloads"]["8 warped pairs 1024x768, K = 2000, AffNet + histogram"] = measure(lafs, lafs, tent, ntent, pairs.tolist(), args)
    gl, gt, gn, gp, H16, _, _, _ = graf_pair((a, o, h))
    Dg = true_frame_distances(gl, gt, gn, gp, [H16])
    Dall = np.concatenate(Dw + Dg)
    keep = {str(c): float((Dall <= c).mean()) for c in CANDIDATES}
    choice = next((c for c in CANDIDATES if keep[str(c)] >= 0.95), None)
    q = [0.5, 0.75, 0.9, 0.95, 0.99]
    res["frame_distance_of_gt_true"] = dict(
        rows=int(len(Dall)), rows_per_pair=[int(len(d)) for d in Dw + Dg], quantiles=dict(zip(map(str, q), np.quantile(Dall, q).tolist())),
        kept_at=keep, kept_at_per_pair=[{str(c): float((d <= c).mean()) for c in CANDIDATES} for d in Dw + Dg],
        smallest_candidate_keeping_95_percent=choice)
    print("D of %d GT-true tentatives: kept %s -> %s" % (len(Dall), keep, choice), file=sys.stderr)
    del lafs, gl
    torch.cuda.empty_cache()

    B, Hh, Ww, K = 16, 768, 1024, 2000
    pipe = DetectDescribePipeline(B, Hh, Ww, a, h, None, num_features=K, do_ori=True)
    lafs, _, desc, cnt = pipe.run(torch.cat([synthetic_image(Hh, Ww, 1234 + i) for i in range(B)]).cuda())
    pipe.check()
    lafs, cnt = lafs.clone(), cnt.clone()
    pl = [(i, j) for i in range(16) for j in range(16) if i != j]
    tent, ntent, _, _ = match_snn_pairs(desc, cnt, pairs=torch.tensor(pl, device="cuda"))
    res["workloads"]["16 x 1024x768 unrelated images, K = 2000, AffNet + histogram, 240 ordered pairs"] = measure(lafs, lafs, tent, ntent,
                                                                                                                  pl, args)
    del pipe
    torch.cuda.empty_cache()

    for out in (0.4, 0.7, 0.85):
        for P in (1, 132, 1024):
            l1, l2, tent, ntent = constructed(P, out)
            pl = [(p, p) for p in range(P)]
            res["workloads"]["constructed n = 1000, %d %% outliers, 5 %% frame outliers, P = %d" % (round(100 * out), P)] = measure(
                l1, l2, tent, ntent, pl, args)
    res["card"]["after"] = card()["nvidia_smi"]
    doc = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(doc + "\n")
    print(doc)


if __name__ == "__main__":
    main()
