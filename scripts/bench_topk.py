"""Step time of the batched pipeline at large top-K budgets (DetectDescribePipeline(large_k=True), ag_pipeline_create_topk), AffNet x 1 +
OriNet + HardNet, on synthetic images:
  * 2 x 1920x1080 at K = 2000 and 10923 (prefilter int(1.5 K) <= 16384: the shared-memory top-K kernels) and K = 20000 (prefilter 30000:
    the global-memory top-K of csrc/topk.cuh), and
  * 1 x 3840x2160 at K = 40000.
Per workload: CUDA-event time of a CUDA-graph replay after warm-up (median of --steps), keypoints per image, launches, and the share of the
top-K kernels (selection and shape filter, old or new) in the device time of one replay under torch.profiler.  The card's name and power
limit are read in the same run.

    python scripts/bench_topk.py [--steps 20] [--warmup 5] [--out profiles/topk_h100.json]

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

WORKLOADS = [("2 x 1920x1080", 2, 1080, 1920, K) for K in (2000, 10923, 20000)] + [("1 x 3840x2160", 1, 2160, 3840, 40000)]
# kernels of the two top-K steps: the shared-memory ones and the global-memory path (key pass, radix select, tile sort, merges, writers)
TOPK_KERNELS = ("select_kernel", "shape_filter_kernel", "topk_select_kernel", "topk_tile_sort_kernel", "topk_merge_kernel",
                "select_topk_write_kernel", "shape_keys_kernel", "shape_topk_write_kernel")


def kernel_table(pipe, imgs):
    """Device time (ms) of one graph replay per kernel name, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pipe.replay(imgs)
        torch.cuda.synchronize()
    table = {}
    for e in prof.events():
        if getattr(e, "device_type", None) is None or "CUDA" not in str(e.device_type):
            continue
        t = table.setdefault(e.name, [0, 0.0])
        t[0] += 1
        t[1] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    return table


def is_topk(name):
    short = name.split("(")[0].split("<")[0].split("::")[-1]
    return short in TOPK_KERNELS


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_topk.py needs a CUDA device")
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.pipeline import DetectDescribePipeline
    from helpers import load_weights, synthetic_image
    W = load_weights()
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    a, o, h = a.eval().cuda(), o.eval().cuda(), h.eval().cuda()
    res = dict(card=card(), pipeline="AffNet x 1 + OriNet + HardNet, large_k=True", steps=args.steps, warmup=args.warmup, runs={})
    for wname, B, H, Wd, K in WORKLOADS:
        imgs = torch.cat([synthetic_image(H, Wd, 1234 + b) for b in range(B)]).cuda()
        pipe = DetectDescribePipeline(B, H, Wd, a, h, o, num_features=K, do_ori=True, large_k=True)
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
        table = kernel_table(pipe, imgs)
        total = sum(v[1] for v in table.values())
        topk = {k: v for k, v in table.items() if is_topk(k)}
        topk_ms = sum(v[1] for v in topk.values())
        med = ms[len(ms) // 2]
        M = int(1.5 * K)
        res["runs"]["%s, K = %d" % (wname, K)] = dict(
            prefilter=M, topk_path="global memory" if M > 16384 else "shared memory", step_ms_median=med, step_ms_min=ms[0],
            step_ms_max=ms[-1], launches=pipe.launches, keypoints_per_image=counts, workspace_gb=round(pipe.ws_bytes / 1e9, 3),
            profiled_device_ms=round(total, 4), topk_ms=round(topk_ms, 4), topk_share=round(topk_ms / total, 4) if total else None,
            topk_kernels_ms={k: dict(launches=v[0], ms=round(v[1], 4)) for k, v in sorted(topk.items(), key=lambda kv: -kv[1][1])})
        print("%-16s K %6d  %8.3f ms  keypoints %s  top-K kernels %.3f ms (%.1f %%)" % (wname, K, med, counts, topk_ms,
                                                                                      100.0 * topk_ms / max(total, 1e-9)), file=sys.stderr)
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
