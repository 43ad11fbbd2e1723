"""Step time of the batched pipeline in the reference's threshold mode (ag_pipeline_create_th; hesaffnet.py's HessianAffine threshold
th = 28.41, no top-K): HesAffNet + HardNet without orientation, with OriNet, and Baumberg x 16 + gradient histogram (hesaffBaum), each on
  * 2 x synthetic 1024x768 (the bench workload's first two images), capacity C = 32768 keypoints per image, and
  * graf img1 + img6 resized to 1024x768, C = 16384 (img6 has more than 8192 keypoints above th).
Per workload: CUDA-event time of a CUDA-graph replay after warm-up (median of --steps), keypoints per image, Mpix/s and keypoints/s, then,
in a separate run, the per-launch table of the library's event profiler (ag_prof_*) summed by kernel, with the share of the keep-all
selection and shape-filter kernels.  The card's name and power limit are read in the same run.

    python scripts/bench_threshold.py [--steps 20] [--warmup 5] [--out FILE.json]

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

TH = 28.41
# name -> (shape estimator, num_Baum_iters, orientation estimator)
MODES = {
    "hesaffnet (AffNet x1, no orientation)": ("affnet", 1, None),
    "hesaffnet + OriNet": ("affnet", 1, "orinet"),
    "hesaffBaum (Baumberg x16 + histogram)": ("baumberg", 16, "histogram"),
}
NEW_KERNELS = ("select_all_mark_kernel", "select_all_chunk_kernel", "select_all_prefix_kernel", "select_all_scatter_kernel",
               "shape_filter_all_kernel")


def workloads():
    import cv2
    from helpers import gold, gray_from_rgb, synthetic_image
    H, Wd = 768, 1024
    syn = torch.cat([synthetic_image(H, Wd, 1234), synthetic_image(H, Wd, 1235)])
    g = [gray_from_rgb(cv2.resize(rgb, (Wd, H), interpolation=cv2.INTER_LINEAR)) for rgb in (gold("graf_full.npz")["rgb"], gold("graf_match.npz")["rgb6"])]
    return {"2 x synthetic 1024x768, C = 32768": (syn, 32768), "graf img1 + img6 at 1024x768, C = 16384": (torch.cat(g), 16384)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_threshold.py needs a CUDA device")
    import affnet_b200._lib as L
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.pipeline import DetectDescribePipeline
    from helpers import load_weights
    W = load_weights()
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    a, o, h = a.eval().cuda(), o.eval().cuda(), h.eval().cuda()
    res = dict(card=card(), th=TH, steps=args.steps, warmup=args.warmup, runs={})
    for wname, (imgs, cap) in workloads().items():
        imgs = imgs.cuda()
        B, _, H, Wd = imgs.shape
        for mname, (shape, iters, ori) in MODES.items():
            pipe = DetectDescribePipeline(B, H, Wd, a if shape == "affnet" else None, h, o if ori == "orinet" else None, num_features=cap,
                                          do_ori=ori is not None, num_Baum_iters=iters, th=TH)
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
            counts = pipe.count.cpu().tolist()
            table = {}
            for kname, kms in L.profile(lambda: pipe.run(imgs)):
                t = table.setdefault(kname, [0, 0.0])
                t[0] += 1
                t[1] += kms
            prof_total = sum(v[1] for v in table.values())
            new_ms = sum(v[1] for k, v in table.items() if k in NEW_KERNELS)
            med = ms[len(ms) // 2]
            res["runs"]["%s | %s" % (mname, wname)] = dict(
                step_ms_median=med, step_ms_min=ms[0], step_ms_max=ms[-1], launches=pipe.launches, keypoints_per_image=counts,
                mpix_per_s=round(B * H * Wd / (med * 1e3), 2), keypoints_per_s=round(sum(counts) / (med * 1e-3)),
                workspace_gb=round(pipe.ws_bytes / 1e9, 3), profiled_ms=round(prof_total, 4), new_kernels_ms=round(new_ms, 4),
                new_kernels_share=round(new_ms / prof_total, 4) if prof_total else None,
                per_kernel_ms={k: dict(launches=v[0], ms=round(v[1], 4)) for k, v in sorted(table.items(), key=lambda kv: -kv[1][1])})
            print("%-40s %-40s %8.3f ms  keypoints %s  new kernels %.1f %%" % (mname, wname, med, counts, 100.0 * new_ms / max(prof_total, 1e-9)),
                  file=sys.stderr)
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
