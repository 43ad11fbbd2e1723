"""Step time of every estimator mode of the batched pipeline (ag_pipeline_create_ex) at the headline workload: 16 x 1024x768 synthetic
images, K = 2000.  Per mode: CUDA-event time of a CUDA-graph replay after warm-up (median of --steps), then, in a separate run, the
per-launch table of the library's event profiler (ag_prof_*) summed by kernel.  The card's name and power limit are read in the same run.

    python scripts/bench_pipeline_modes.py [--steps 20] [--warmup 5] [--batch 16] [--out FILE.json]

Needs an H100 (there is no CPU path); prints one JSON document.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

# name -> (shape estimator, num_Baum_iters, orientation estimator): "affnet" / "baumberg" / None, "orinet" / "histogram" / None
MODES = {
    "affnet1-orinet (default)": ("affnet", 1, "orinet"),
    "affnet1-histogram": ("affnet", 1, "histogram"),
    "affnet2-orinet": ("affnet", 2, "orinet"),
    "baumberg16-histogram": ("baumberg", 16, "histogram"),
    "baumberg1-none": ("baumberg", 1, None),
    "none-histogram": (None, 0, "histogram"),
    "none-orinet": (None, 0, "orinet"),
    "none-none": (None, 0, None),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return dict(name=torch.cuda.get_device_name(), nvidia_smi=q)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pipeline_modes.py needs a CUDA device")
    import affnet_b200._lib as L
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.pipeline import DetectDescribePipeline
    from helpers import load_weights, synthetic_image
    W = load_weights()
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    a, o, h = a.eval().cuda(), o.eval().cuda(), h.eval().cuda()
    B, H, Wd, K = args.batch, 768, 1024, 2000
    imgs = torch.cat([synthetic_image(H, Wd, 1234 + i) for i in range(B)]).cuda()
    res = dict(card=card(), workload="%d x %dx%d synthetic, K = %d" % (B, Wd, H, K), steps=args.steps, warmup=args.warmup, modes={})
    for name, (shape, iters, ori) in MODES.items():
        pipe = DetectDescribePipeline(B, H, Wd, a if shape == "affnet" else None, h, o if ori == "orinet" else None, num_features=K,
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
        counts = pipe.count.cpu().tolist()
        table = {}
        for kname, kms in L.profile(lambda: pipe.run(imgs)):
            t = table.setdefault(kname, [0, 0.0])
            t[0] += 1
            t[1] += kms
        res["modes"][name] = dict(step_ms_median=ms[len(ms) // 2], step_ms_min=ms[0], step_ms_max=ms[-1], launches=pipe.launches,
                                  keypoints_per_image_min=min(counts), keypoints_per_image_max=max(counts),
                                  per_kernel_ms={k: dict(launches=v[0], ms=round(v[1], 4)) for k, v in sorted(table.items(), key=lambda kv: -kv[1][1])})
        print("%-26s %8.3f ms (min %.3f, max %.3f)  %d launches" % (name, ms[len(ms) // 2], ms[0], ms[-1], pipe.launches), file=sys.stderr)
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
