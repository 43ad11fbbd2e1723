"""SIFT descriptor cost at the headline workload: 16 x 1024x768 synthetic images, K = 2000 (32,000 keypoints).

  - Kernel time of the fused descriptor stage (sift_pyr_kernel = ag_sift_describe_pyr) inside the AffNet + histogram pipeline at
    PS 32, 41 and 65: the library's event profiler (ag_prof_*), median over --steps runs.
  - Step time (CUDA-event time of a CUDA-graph replay after warm-up, median of --steps) of AffNet x1 + OriNet, Baumberg x16 + histogram
    and none + histogram, each with HardNet and with SIFT(32), and the per-kernel table of one profiled run.
The card's name and power limit are read in the same run.

    python scripts/bench_sift.py [--steps 20] [--warmup 5] [--batch 16] [--out FILE.json]

Needs an H100 (there is no CPU path); prints one JSON document.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from bench_pipeline_modes import card  # noqa: E402

MODES = {
    "affnet1-orinet": ("affnet", 1, "orinet"),
    "baumberg16-histogram": ("baumberg", 16, "histogram"),
    "none-histogram": (None, 0, "histogram"),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sift.py needs a CUDA device")
    import affnet_b200._lib as L
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.pytorch_sift import SIFTNet
    from helpers import load_weights, synthetic_image
    W = load_weights()
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    a, o, h = a.eval().cuda(), o.eval().cuda(), h.eval().cuda()
    B, H, Wd, K = args.batch, 768, 1024, 2000
    imgs = torch.cat([synthetic_image(H, Wd, 1234 + i) for i in range(B)]).cuda()
    res = dict(card=card(), workload="%d x %dx%d synthetic, K = %d" % (B, Wd, H, K), steps=args.steps, warmup=args.warmup,
               sift_kernel={}, modes={})

    def profiled(pipe):
        table = {}
        for kname, kms in L.profile(lambda: pipe.run(imgs)):
            t = table.setdefault(kname, [0, 0.0])
            t[0] += 1
            t[1] += kms
        return table

    for PS in (32, 41, 65):
        pipe = DetectDescribePipeline(B, H, Wd, a, SIFTNet(PS), None, num_features=K, do_ori=True)
        for _ in range(args.warmup):
            pipe.run(imgs)
        ms = sorted(profiled(pipe)["sift_pyr_kernel"][1] for _ in range(args.steps))
        pipe.check()
        n = int(pipe.count.sum())
        res["sift_kernel"]["PS %d" % PS] = dict(ms_median=ms[len(ms) // 2], ms_min=ms[0], ms_max=ms[-1], keypoints=n)
        print("sift_pyr_kernel PS %d: %.3f ms (min %.3f, max %.3f), %d keypoints" % (PS, ms[len(ms) // 2], ms[0], ms[-1], n), file=sys.stderr)
        del pipe
    for name, (shape, iters, ori) in MODES.items():
        for dname, desc in (("hardnet", h), ("sift32", SIFTNet(32))):
            pipe = DetectDescribePipeline(B, H, Wd, a if shape == "affnet" else None, desc, o if ori == "orinet" else None, num_features=K,
                                          do_ori=ori is not None, num_Baum_iters=iters)
            pipe.capture()
            for _ in range(args.warmup):
                pipe.replay(imgs)
            torch.cuda.synchronize()
            ms = []
            for _ in range(args.steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                pipe.replay(imgs)
                e1.record()
                e1.synchronize()
                ms.append(e0.elapsed_time(e1))
            ms.sort()
            pipe.check()
            table = profiled(pipe)
            res["modes"]["%s + %s" % (name, dname)] = dict(
                step_ms_median=ms[len(ms) // 2], step_ms_min=ms[0], step_ms_max=ms[-1], launches=pipe.launches, workspace_bytes=pipe.ws_bytes,
                per_kernel_ms={k: dict(launches=v[0], ms=round(v[1], 4)) for k, v in sorted(table.items(), key=lambda kv: -kv[1][1])})
            print("%-34s %8.3f ms (min %.3f, max %.3f)  %d launches" % ("%s + %s" % (name, dname), ms[len(ms) // 2], ms[0], ms[-1],
                                                                       pipe.launches), file=sys.stderr)
            del pipe
            torch.cuda.empty_cache()
    res["card"]["after"] = card()["nvidia_smi"]
    doc = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(doc + "\n")
    print(doc)


if __name__ == "__main__":
    main()
