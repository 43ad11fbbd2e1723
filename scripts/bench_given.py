"""Step time of the given-keypoints pipeline (ag_pipeline_create_given, DescribeGivenPipeline): AffNet x 1 + OriNet + HardNet on
B = 16 synthetic 1024x768 images (the bench workload's images) with C = 2000 upright keypoints per image - the detector's own top-2000
without a shape or orientation step - and, on the same images, the detect pipeline's step (AffNet x 1 + OriNet + HardNet, K = 2000) for
comparison.  Per pipeline: CUDA-event time of a CUDA-graph replay after warm-up (median of --steps), then, in a separate run, the device
time of the replayed kernels from torch.profiler, summed by kernel.  The card's name and power limit are read in the same run.

    python scripts/bench_given.py [--steps 20] [--warmup 5] [--out profiles/given_h100.json]

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

B, H, W, C = 16, 768, 1024, 2000


def timed(replay, steps, warmup):
    for _ in range(warmup):
        replay()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        replay()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    ms.sort()
    return dict(step_ms_median=ms[len(ms) // 2], step_ms_min=ms[0], step_ms_max=ms[-1])


def device_time(replay, reps=5):
    """torch.profiler over `reps` graph replays: the kernels' device time per step, in total and by kernel name."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            replay()
        torch.cuda.synchronize()
    table = {}
    for e in prof.events():
        if e.device_type != DeviceType.CUDA:
            continue
        t = table.setdefault(e.name, [0, 0.0])
        t[0] += 1
        t[1] += e.time_range.elapsed_us() / 1e3
    total = sum(v[1] for v in table.values()) / reps
    top = sorted(table.items(), key=lambda kv: -kv[1][1])[:12]
    return dict(device_ms_per_step=round(total, 4),
                top_kernels_ms_per_step={k: dict(launches_per_step=v[0] / reps, ms=round(v[1] / reps, 4)) for k, v in top})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_given.py needs a CUDA device")
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.pipeline import DescribeGivenPipeline, DetectDescribePipeline
    from helpers import load_weights, synthetic_image
    Wt = load_weights()
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(Wt["affnet"]); o.load_state_dict(Wt["orinet"]); h.load_state_dict(Wt["hardnet"])
    a, o, h = a.eval().cuda(), o.eval().cuda(), h.eval().cuda()
    res = dict(card=card(), workload="B = %d x %dx%d synthetic, C = %d upright keypoints per image, AffNet x1 + OriNet + HardNet" % (B, W, H, C),
               steps=args.steps, warmup=args.warmup, runs={})
    imgs = torch.cat([synthetic_image(H, W, 1234 + i) for i in range(B)]).cuda().contiguous()
    plain = DetectDescribePipeline(B, H, W, None, h, None, num_features=C, do_ori=False, num_Baum_iters=0)
    lafs, _, _, cnt = plain.run(imgs)
    lafs, cnt = lafs.clone(), cnt.clone()
    torch.cuda.synchronize()
    del plain
    torch.cuda.empty_cache()

    given = DescribeGivenPipeline(B, H, W, a, h, o, capacity=C, do_ori=True, num_Baum_iters=1).capture()
    given.replay(imgs, lafs, cnt)
    r = timed(lambda: given.replay(), args.steps, args.warmup)
    r.update(device_time(lambda: given.replay()), launches=given.launches, keypoints_in=cnt.cpu().tolist(),
             survivors=given.count.cpu().tolist(), workspace_gb=round(given.ws_bytes / 1e9, 3))
    r["keypoints_per_s"] = round(sum(r["survivors"]) / (r["step_ms_median"] * 1e-3))
    res["runs"]["given keypoints (ag_pipeline_run_given)"] = r
    print("given   %8.3f ms median, device %.3f ms, %d launches" % (r["step_ms_median"], r["device_ms_per_step"], r["launches"]), file=sys.stderr)
    del given
    torch.cuda.empty_cache()

    det = DetectDescribePipeline(B, H, W, a, h, o, num_features=C, do_ori=True, num_Baum_iters=1).capture()
    r = timed(lambda: det.replay(imgs), args.steps, args.warmup)
    r.update(device_time(lambda: det.replay(imgs)), launches=det.launches, keypoints=det.count.cpu().tolist(),
             workspace_gb=round(det.ws_bytes / 1e9, 3))
    res["runs"]["detect and describe (ag_pipeline_run), same images"] = r
    print("detect  %8.3f ms median, device %.3f ms, %d launches" % (r["step_ms_median"], r["device_ms_per_step"], r["launches"]), file=sys.stderr)
    res["card"]["after"] = card()["nvidia_smi"]
    doc = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(doc + "\n")
    print(doc)


if __name__ == "__main__":
    main()
