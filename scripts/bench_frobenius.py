"""Device Frobenius ground truth (ReprojectionStuff.frobenius_gt_sets / frobenius_gt_pairs, the reference's
get_GT_correspondence_indexes_Fro criterion; default flags, dist_threshold 4).  Workloads:
  - set mode on 8 pipeline pairs of 16 synthetic 1024x768 images, K = 2000 (whole detection sets: repeatability);
  - tentative mode on the same pairs after match_snn_pairs;
  - set mode on the 240 ordered pairs of the 16 images;
  - one 20000 x 20000 set-mode pair of random frames.
Device: CUDA-event time of a CUDA-graph replay of the call alone (median of --steps after --warmup, --rounds times).  The kernels' share
of the FP32 bound uses OPS_PER_PAIR fp32 operations per (row, column) of the default variant (frob_scan<INV, !SKIP, !GATE>) over the
H100 SXM data sheet's 67 TFLOP/s.  Also: the numpy restatement's time for one 2000 x 2000 pair on the host CPU (labelled, for
comparison), and, informational, graf 1 -> 6 affine-region repeatability at K = 2000 for the plain detector, HesAff (Baumberg x 16) and
HesAffNet.  The card's name and power limit are read in the same run.
    python scripts/bench_frobenius.py [--steps 20] [--warmup 5] [--rounds 2] [--out FILE.json]
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

# M = B A' (8 mul, 4 add), two subtractions of 1, the four squares summed (4 mul, 3 add), r = B t' + c (4 mul, 4 add), |r|^2 added
# (2 mul, 2 add): 33 roundings, plus the comparison with the running minimum (not counted)
OPS_PER_PAIR = 33
FP32_PEAK = 67e12


def timed(fn, args, work):
    res = []
    out = None
    for _ in range(args.rounds):
        t, out = graph_ms(fn, args.steps, args.warmup)
        res.append(t)
    med = sorted(t["median"] for t in res)[0]
    r = dict(graph_ms=res, best_median_ms=med, row_column_pairs=work, fp32_ops=work * OPS_PER_PAIR)
    r["fp32_bound_ms"] = work * OPS_PER_PAIR / FP32_PEAK * 1e3
    r["share_of_fp32_bound"] = r["fp32_bound_ms"] / med
    print("%-60s %9.3f ms  %.2f of the FP32 bound" % (fn.__name__ if hasattr(fn, "__name__") else "", med, r["share_of_fp32_bound"]),
          file=sys.stderr)
    return r, out


def random_frames(g, n):
    s = np.exp(g.uniform(0.5, 3.0, n))
    ang = g.uniform(0, 2 * np.pi, n)
    c, si = np.cos(ang), np.sin(ang)
    a = np.stack([np.stack([s * c, -s * si], 1), np.stack([s * si, s * c], 1)], 1)
    return np.concatenate([a, g.uniform(0, 2000, (n, 2, 1))], 2).astype(np.float32)


def repeatability(nets):
    """graf img1 -> img6 with H1to6, K = 2000: rows of img1 whose Frobenius-nearest img6 frame is within dist_threshold 4 (with and
    without the reference's centre and scale gates), over min(n1, n6)."""
    from affnet_b200.HandCraftedModules import AffineShapeEstimator
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.ReprojectionStuff import frobenius_gt_sets
    from helpers import gold, gray_from_rgb
    a, h = nets
    z, m = gold("graf_full.npz"), gold("graf_match.npz")
    imgs = torch.cat([gray_from_rgb(z["rgb"]), gray_from_rgb(m["rgb6"])]).cuda()
    H = torch.from_numpy(m["H1to6"]).float().cuda()
    out = {}
    for name, shape, iters in (("plain detector", a, 0), ("HesAff (Baumberg x 16)", AffineShapeEstimator(19).cuda(), 16),
                               ("HesAffNet", a, 1)):
        pipe = DetectDescribePipeline(2, imgs.size(2), imgs.size(3), shape, h, None, num_features=2000, do_ori=False, num_Baum_iters=iters)
        lafs, _, _, cnt = pipe.run(imgs)
        n1, n6 = cnt.tolist()
        pairs = torch.tensor([[0, 1]], device="cuda")
        r = dict(n1=n1, n6=n6)
        for crit, kw in (("Fro", {}), ("Fro_and_center", dict(center_dist_th=2.0))):
            _, ntrue, _, _ = frobenius_gt_sets(lafs, cnt, H, pairs=pairs, **kw)
            r[crit] = dict(true=int(ntrue[0]), repeatability=int(ntrue[0]) / max(min(n1, n6), 1))
        out[name] = r
        del pipe
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frobenius.py needs a CUDA device")
    import frobenius_restated as FR
    from affnet_b200.architectures import AffNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.ReprojectionStuff import frobenius_gt_pairs, frobenius_gt_sets
    from helpers import load_weights, synthetic_image
    W = load_weights()
    a, h = AffNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); h.load_state_dict(W["hardnet"])
    a, h = a.eval().cuda(), h.eval().cuda()
    res = dict(card=card(), steps=args.steps, warmup=args.warmup, rounds=args.rounds, ops_per_row_column=OPS_PER_PAIR,
               fp32_peak_flops=FP32_PEAK, workloads={})

    B, Hh, Ww, K = 16, 768, 1024, 2000
    pipe = DetectDescribePipeline(B, Hh, Ww, a, h, None, num_features=K, do_ori=False)
    lafs, _, desc, cnt = pipe.run(torch.cat([synthetic_image(Hh, Ww, 1234 + i) for i in range(B)]).cuda())
    lafs, desc, cnt = lafs.clone(), desc.clone(), cnt.clone()
    del pipe
    torch.cuda.empty_cache()
    c = cnt.tolist()
    for pname, pl in (("8 pairs", [(2 * k, 2 * k + 1) for k in range(8)]),
                      ("240 ordered pairs", [(i, j) for i in range(B) for j in range(B) if i != j])):
        pairs = torch.tensor(pl, device="cuda")
        Hid = torch.eye(3, device="cuda").expand(len(pl), 3, 3).contiguous()
        work = sum(c[i] * c[j] for i, j in pl)
        r, out = timed(lambda: frobenius_gt_sets(lafs, cnt, Hid, pairs=pairs), args, work)
        r["true_rows"] = out[1].tolist()
        res["workloads"]["set mode, %s of 16 x 1024x768, K = 2000" % pname] = r
        if pname == "8 pairs":
            tent, ntent, _, _ = match_snn_pairs(desc, cnt, pairs=pairs)
            nt = ntent.tolist()
            r, out = timed(lambda: frobenius_gt_pairs(lafs, tent, ntent, Hid, pairs=pairs), args, sum(n * n for n in nt))
            r.update(tentatives=nt, true_rows=out[1].tolist())
            res["workloads"]["tentative mode, 8 pairs after match_snn_pairs"] = r

    g = np.random.default_rng(3)
    n = 20000
    l1 = torch.from_numpy(random_frames(g, n)).cuda()[None]
    l2 = torch.from_numpy(random_frames(g, n)).cuda()[None]
    cn = torch.tensor([n], dtype=torch.int32, device="cuda")
    H = torch.eye(3, device="cuda")
    r, _ = timed(lambda: frobenius_gt_sets(l1, cn, H, l2, cn), args, n * n)
    res["workloads"]["set mode, one 20000 x 20000 pair"] = r

    g = np.random.default_rng(4)
    c1, c2 = random_frames(g, 2000), random_frames(g, 2000)
    prm = FR.Params()
    ms = []
    for _ in range(3):
        t0 = time.perf_counter()
        FR.frobenius(c1, c2, np.eye(3, dtype=np.float32), prm)
        ms.append((time.perf_counter() - t0) * 1e3)
    res["cpu_restatement_2000x2000_ms"] = dict(median=sorted(ms)[1], label="numpy restatement on the host CPU (%d threads), for comparison"
                                               % torch.get_num_threads())
    res["graf_1_to_6_repeatability_K2000"] = repeatability((a, h))
    s = json.dumps(res, indent=1)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")
    print(s)


if __name__ == "__main__":
    main()
